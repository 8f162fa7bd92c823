// stage.cu - the stage runtime behind the C-ABI (include/defer_b200.h).
//
// A stage is what one reference compute node holds after `model_from_json` + `set_weights`
// (src/node.py:31-38) and runs in its `_data_client` loop (src/node.py:103-108).  Here it is:
//   * weights resident in HBM (bias+BN folded by the host planner into per-channel scale/shift),
//   * `depth` lanes; each lane = stream + activation workspace + one CUDA graph of the fused-op chain,
//   * an exported arena [ctrl flags | input slots] that the upstream stage writes over NVLink.
// Microbatch k runs on lane k % depth at every stage, so compute of k overlaps the hop of k-1 and
// the arrival of k+1 (double buffering when depth == 2).
#include <stdarg.h>
#include <string.h>
#include <unistd.h>

#include <mutex>
#include <algorithm>
#include <set>
#include <utility>
#include <stdlib.h>
#include <string>
#include <vector>

#include "common.cuh"
#include "conv_umma.cuh"

namespace defer {

// ------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

void prefer_max_smem_impl(const void* func) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return;
  std::lock_guard<std::mutex> lk(mu);
  if (done.count({func, dev})) return;
  if (getenv("DEFER_NO_CARVEOUT") == nullptr)
    cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaGetLastError();
  done.insert({func, dev});
}

// ------------------------------------------------------------------------------------------ layout
constexpr int MAX_DEPTH = 32;
constexpr size_t CTRL_BYTES = 16384;
constexpr size_t FLAG_STRIDE = 128;  // one flag per 128-B line
// ctrl block: [0,4096) ready[d] | [4096,8192) free[d] | [8192,..) local counters | status
constexpr size_t OFF_READY = 0, OFF_FREE = 4096, OFF_CTR = 8192, OFF_STATUS = 12288;
enum { CTR_WAIT_READY = 0, CTR_SIG_FREE = 1, CTR_WAIT_FREE = 2, CTR_SIG_READY = 3 };

struct LinkToken {  // POD, <= DEFER_LINK_TOKEN_BYTES
  uint32_t magic;
  int32_t role;
  int32_t device;
  int32_t pid;
  int32_t depth;
  int32_t fmt;
  int32_t batch;
  uint64_t slot_bytes;     // bytes of one input slot (role 0)
  uint64_t arena_bytes;
  uint64_t off_slots;      // offset of slot 0 in the arena
  uint64_t slot_stride;
  uint64_t local_base;     // arena base in the exporting process (same-pid import)
  cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(LinkToken) <= DEFER_LINK_TOKEN_BYTES, "token too large");
constexpr uint32_t TOKEN_MAGIC = 0xDEFE7B20u;

struct Buf {
  int h, w, c, elem;
  size_t elems;  // per microbatch
  size_t bytes;
};

struct OpRt {
  defer_op_desc d;
  int backend = 1;          // 1 SIMT, 2 wgmma, 4 tensor-core stem (im2col of the fp32 image + wgmma 1x1 conv)
  int k_pad = 0;            // backend 4: padded patch length (multiple of 64)
  void* w_pad = nullptr;    // backend 4: zero-padded [k_pad, cout] fp32 filter matrix
  bool persist = false;     // wgmma conv with many tiles: persistent-grid launch (overlapped epilogue)
  bool stem_fused = false;  // backend 4 without a patch matrix: conv_stem_kernel builds the A operand from the fp32 image
  bool stream = false;      // ... with the plan's N tile (64 | 128); false = the 64-wide persistent grid (DEFER_STREAM=0, launch_conv_persistent)
  int n_tiles64 = 0;
  int stem_tiles = 0;       // fused stem: 2-D output tiles it launches over (umma_mega_set_stem)
  UmmaConvPlan umma;        // valid when backend == 2
  std::string kname;
  double alg_bytes = 0, alg_flops = 0;
  int n_kernels = 1;
  // Keras preprocessing (DEFER_OP_PREPROCESS, caffe or tf mode).  It is folded into the fused stem conv that reads its output when
  // that conv is its only reader; the op then launches nothing and its F32 image is never written.
  float pre_shift[3] = {0.f, 0.f, 0.f};   // PREPROCESS, caffe: host copy of the shift weights (tf has none)
  int folded_into = -1;                   // PREPROCESS / AFFINE: index of the conv that applies it, -1 = runs its own kernel
  int u8_pre = -1;                        // fused stem conv: index of the PREPROCESS op folded into it, -1 = none
  // A standalone AFFINE(+ReLU) that reads a wgmma conv's output is folded into that conv's epilogue (DEFER_FOLD_AFFINE=1):
  // the conv writes the affine op's output too, and its own output only when something else reads it.
  int aff_op = -1;                        // wgmma conv: index of the AFFINE op folded into it, -1 = none
  bool store_out = true;                  // ... false: the conv's own output buffer is never written
};

struct Lane {
  cudaStream_t stream = nullptr;
  std::vector<void*> buf;   // device pointer per plan buffer
  cudaGraphExec_t exec = nullptr;
  cudaGraph_t graph = nullptr;
  cudaEvent_t done = nullptr, t0 = nullptr, t1 = nullptr, join = nullptr;
  float* out_host = nullptr;  // pinned, last stage
  int* status_host = nullptr; // pinned copy of the sticky device status, refreshed every step (last stage)
  float* dense_partial = nullptr;
  std::vector<UmmaConvLaneArgs> umma;  // per op
  std::vector<void*> persist_op;       // per op: device op descriptor for the persistent-grid launch
  std::vector<void*> im2col;           // per op (backend 4): patch matrix scratch
  bool timed = false;
  void* peer_out = nullptr;   // HOP_COPY: this lane's input slot on the consumer GPU (destination of the hop copy)
  int32_t* tables = nullptr;  // DEFER_RESIZE_SAMPLE_*: `batch` table blocks, next to the lane's input slot in the arena
  int32_t* dec_blocks = nullptr;   // DEFER_OP_JPEG_DECODE / _PNG_DECODE / _IMAGE_DECODE: `batch` blocks, after the table blocks
  void* dec_ws = nullptr;          // ... and its decode workspace
  // the microbatch the lane ran last (last stage: the one out_host is filled with); result() refuses any other
  bool stepped = false;
  uint64_t last_seq = 0;
};

// How a non-last stage's output reaches the next GPU's input slot (DEFER_HOP, read when the stage is created):
//   HOP_COPY   (default) the last op writes a LOCAL buffer; then the lane waits for the
//              slot's free flag and a cudaMemcpyAsync (copy engine, captured in the lane graph) ships it over NVLink in
//              full-line bursts - the north star's cudaMemcpyPeerAsync hop.  Compute never blocks on back-pressure and no
//              SM spends time on small peer stores.
//   HOP_TMA    the last op's epilogue stores into the peer slot directly (same stores as HOP_DIRECT on this kernel).
//   HOP_DIRECT per-thread st.global of the epilogue into the peer slot.
enum HopMode { HOP_COPY = 0, HOP_TMA = 1, HOP_DIRECT = 2 };

struct Mark {                 // steady-state timing: an event recorded right behind one chosen microbatch
  cudaEvent_t ev = nullptr;
  bool recorded = false;
};

}  // namespace defer

using namespace defer;

struct defer_stage_s {
  defer_stage_config cfg;
  std::vector<Buf> bufs;
  std::vector<OpRt> ops;
  std::vector<void*> d_weights;        // fp32 device copies, by weight id
  std::vector<size_t> weight_bytes;
  std::vector<void*> d_weights_bf16;   // dense kernels in bf16 (fmt == BF16) or null
  std::vector<Lane> lanes;
  uint8_t* arena = nullptr;            // [ctrl | input slots]
  size_t arena_bytes = 0, slot_stride = 0;
  std::vector<void*> workspace;        // everything else we cudaMalloc'ed
  // links
  bool has_prod = false, has_cons = false, finalized = false, unlinked = false;
  uint8_t* cons_arena = nullptr;       // consumer arena mapped here (slots + ready flags)
  size_t cons_off_slots = 0, cons_slot_stride = 0;
  uint8_t* prod_arena = nullptr;       // producer arena mapped here (free flags)
  bool cons_is_ipc = false, prod_is_ipc = false;
  int last_input_reader = -1, output_writer = -1;
  unsigned long long timeout_ns = 4000ull * 1000000ull;
  void* flush_buf = nullptr;
  size_t flush_bytes = 0;
  size_t max_dense_partial = 0;
  cudaEvent_t job_t0 = nullptr, job_t1 = nullptr;
  Mark marks[2];
  int hop = HOP_COPY;
  // megakernel groups: runs of consecutive wgmma convs executed by one cluster launch per lane
  struct MegaGroup {
    int first = 0, last = 0;
    std::vector<void*> dev_ops;   // per lane: device array of op descriptors
  };
  std::vector<MegaGroup> groups;
  std::vector<int> op_group;      // group index per op, -1 = launched on its own
  // images of mixed sizes: the DEFER_RESIZE_SAMPLE_W / _H pair (op indices, -1 = none), its geometry and table blocks
  struct Frames {
    int op_w = -1, op_h = -1;
    int H = 0, W = 0, H_out = 0, W_out = 0, kw_w = 0, kw_h = 0;
    size_t block_ints = 0;        // int32 values per sample block
    size_t tables_off = 0;        // offset of a lane's blocks from its input slot
  } frames;
  // JPEG or PNG files at ingress: the DEFER_OP_JPEG_DECODE, _PNG_DECODE or _IMAGE_DECODE op (-1 = none) in front of the
  // per-sample resize pair
  struct Decode {
    int op = -1;
    int kind = 0;                 // its op kind
    size_t block_ints = 0;        // DEFER_JPEG_BLOCK_INTS, DEFER_PNG_BLOCK_INTS or DEFER_IMAGE_BLOCK_INTS
    size_t blocks_off = 0;        // offset of a lane's blocks from its input slot
    size_t ws_bytes = 0;          // decode workspace per lane
  } dec;

  uint32_t* ctrl_u32(size_t off) { return reinterpret_cast<uint32_t*>(arena + off); }
  uint32_t* ready_flag(int d) { return ctrl_u32(OFF_READY + d * FLAG_STRIDE); }
  uint32_t* free_flag(int d) { return ctrl_u32(OFF_FREE + d * FLAG_STRIDE); }
  uint32_t* counter(int which, int d) { return ctrl_u32(OFF_CTR + (which * MAX_DEPTH + d) * 4); }
  int* status_ptr() { return reinterpret_cast<int*>(arena + OFF_STATUS); }
};

namespace defer {

static size_t elem_bytes(int elem, int fmt) {
  const bool bytes = elem == DEFER_BUF_U8 || elem == DEFER_BUF_JPEG || elem == DEFER_BUF_PNG || elem == DEFER_BUF_IMAGE;
  return bytes ? 1 : elem == DEFER_BUF_F32 ? 4 : fmt_bytes_per_elem(fmt);
}

static size_t buf_bytes(const Buf& b, int fmt) { return b.elems * elem_bytes(b.elem, fmt); }

// the files a stage with a decode op takes, for messages: "JPEG" / "jpeg", "PNG" / "png" or "JPEG or PNG" / "image"
static const char* dec_name(const defer_stage_s* s, bool upper) {
  if (s->dec.kind == DEFER_OP_IMAGE_DECODE) return upper ? "JPEG or PNG" : "image";
  return s->dec.kind == DEFER_OP_PNG_DECODE ? (upper ? "PNG" : "png") : (upper ? "JPEG" : "jpeg");
}

// the axis of a fixed-table RESIZE op: named by modes W / H (it may keep its length under a crop box), else the one that
// changes
static bool resize_horizontal(const defer_op_desc& d, const Buf& bi, const Buf& bo) {
  return d.mode == DEFER_RESIZE_W || (d.mode == 0 && bi.w != bo.w);
}

static int set_device(const defer_stage_s* s) {
  DEFER_CUDA(cudaSetDevice(s->cfg.device));
  return DEFER_OK;
}

// ------------------------------------------------------------------------------------------ op launch
static int launch_op(defer_stage_s* s, int lane_id, int oi, cudaStream_t st) {
  Lane& L = s->lanes[lane_id];
  OpRt& op = s->ops[oi];
  const defer_op_desc& d = op.d;
  const int fmt = s->cfg.fmt, nb = s->cfg.batch;
  const Buf& bi = s->bufs[d.in0];
  const Buf& bo = s->bufs[d.out];
  void* x = L.buf[d.in0];
  void* y = L.buf[d.out];
  auto wptr = [&](int id) -> const float* { return id >= 0 ? (const float*)s->d_weights[id] : nullptr; };
  switch (d.kind) {
    case DEFER_OP_CONV: {
      if (op.backend == 4 && op.stem_fused)
        return launch_conv_stem(op.umma.nplanes, L.persist_op[oi], op.stem_tiles, op.u8_pre >= 0,
                                op.u8_pre >= 0 && s->ops[op.u8_pre].d.mode == DEFER_PRE_TF, st);
      if (op.backend == 4)
        DEFER_TRY(launch_stem_im2col(fmt, (const float*)x, L.im2col[oi], nb, bi.h, bi.w, bi.c, d.kh, d.kw, d.sh, d.sw, d.pad_t,
                                     d.pad_l, bo.h, bo.w, op.k_pad, st));
      if (op.backend == 2 || op.backend == 4) {
        if (op.stream)
          return launch_conv_stream(op.umma.nplanes, op.umma.bn, L.persist_op[oi],
                                    op.umma.m_tiles * (op.umma.cout / op.umma.bn),
                                    op.umma.k_blocks, op.aff_op >= 0, st);
        if (op.persist) return launch_conv_persistent(op.umma.nplanes, L.persist_op[oi], op.n_tiles64, op.aff_op >= 0, st);
        return launch_conv_umma(op.umma, L.umma[oi], st);
      }
      ConvParams p;
      p.x = x; p.w = wptr(d.w_kernel); p.scale = wptr(d.w_scale); p.shift = wptr(d.w_shift);
      p.res = (d.flags & DEFER_FLAG_RESIDUAL) ? L.buf[d.in1] : nullptr;
      p.y = y;
      p.n = nb; p.h = bi.h; p.w_in = bi.w; p.cin = bi.c;
      p.ho = bo.h; p.wo = bo.w; p.cout = bo.c;
      p.kh = d.kh; p.kw = d.kw; p.sh = d.sh; p.sw = d.sw; p.pad_t = d.pad_t; p.pad_l = d.pad_l;
      p.flags = d.flags;
      return launch_conv_simt(fmt, bi.elem == DEFER_BUF_F32, p, st);
    }
    case DEFER_OP_MAXPOOL:
      return launch_maxpool(fmt, x, y, nb, bi.h, bi.w, bi.c, d.kh, d.kw, d.sh, d.sw, d.pad_t, d.pad_l, bo.h, bo.w, st);
    case DEFER_OP_GAP:
      return launch_gap(fmt, x, y, nb, bi.h, bi.w, bi.c, st);
    case DEFER_OP_DENSE: {
      int F = bi.h * bi.w * bi.c, U = bo.c;
      bool wb = s->d_weights_bf16[d.w_kernel] != nullptr;
      const void* w = wb ? s->d_weights_bf16[d.w_kernel] : s->d_weights[d.w_kernel];
      return launch_dense(fmt, x, w, wb, wptr(d.w_shift), y, bo.elem == DEFER_BUF_F32, L.dense_partial, nb, F, U,
                          d.flags, st);
    }
    case DEFER_OP_SOFTMAX:
      return launch_softmax((const float*)x, (float*)y, nb, bo.c, st);
    case DEFER_OP_AFFINE:
      if (op.folded_into >= 0) return DEFER_OK;   // written by the conv's epilogue
      [[fallthrough]];
    case DEFER_OP_RELU:
    case DEFER_OP_ADD:
      return launch_eltwise(fmt, d.kind, x, d.in1 >= 0 ? L.buf[d.in1] : nullptr, wptr(d.w_scale), wptr(d.w_shift), y,
                            (size_t)nb * bi.h * bi.w, bi.c, d.flags, st);
    case DEFER_OP_PAD:
      return launch_pad(fmt, x, y, nb, bi.h, bi.w, bi.c, d.pad_t, d.pad_l, bo.h, bo.w, st);
    case DEFER_OP_COPY:
      if (bi.elem == bo.elem) {
        if (bi.elem == DEFER_BUF_F32) {
          DEFER_CUDA(cudaMemcpyAsync(y, x, bi.elems * 4, cudaMemcpyDeviceToDevice, st));
          return DEFER_OK;
        }
        return launch_copy_act(fmt, x, y, bi.elems, st);
      }
      if (bi.elem == DEFER_BUF_F32) return launch_encode(fmt, (const float*)x, y, bi.elems, st);
      return launch_decode(fmt, x, (float*)y, bi.elems, st);
    case DEFER_OP_PREPROCESS:
      if (op.folded_into >= 0) return DEFER_OK;   // applied by the stem conv as it reads the image
      if (d.mode == DEFER_PRE_TF) return launch_preprocess_tf((const uint8_t*)x, (float*)y, (size_t)nb * bi.h * bi.w, st);
      return launch_preprocess((const uint8_t*)x, wptr(d.w_shift), (float*)y, (size_t)nb * bi.h * bi.w, st);
    case DEFER_OP_JPEG_DECODE:
      return launch_jpeg_decode((const uint8_t*)x, L.dec_blocks, nb, bi.h, bi.w, L.dec_ws, (uint8_t*)y, st);
    case DEFER_OP_PNG_DECODE:
      return launch_png_decode((const uint8_t*)x, L.dec_blocks, nb, bi.h, bi.w, L.dec_ws, (uint8_t*)y, st);
    case DEFER_OP_IMAGE_DECODE:
      return launch_image_decode((const uint8_t*)x, L.dec_blocks, nb, bi.h, bi.w, L.dec_ws, (uint8_t*)y, st);
    case DEFER_OP_RESIZE:
      if (d.mode == DEFER_RESIZE_SAMPLE_W || d.mode == DEFER_RESIZE_SAMPLE_H) {
        const auto& f = s->frames;
        return launch_resize_frames(d.mode, (const uint8_t*)x, (uint8_t*)y, L.tables, nb, f.H, f.W, f.H_out, f.W_out, f.kw_w,
                                    f.kw_h, st);
      }
      return launch_resize((const uint8_t*)x, (uint8_t*)y, (const int32_t*)s->d_weights[d.w_scale],
                           (const int32_t*)s->d_weights[d.w_kernel], d.kw, nb, bi.h, bi.w, bo.h, bo.w,
                           resize_horizontal(d, bi, bo), st);
  }
  set_error("launch_op: unknown op kind %d", d.kind);
  return DEFER_ERR_INVALID;
}

// enqueue one microbatch worth of work on a lane (captured into the lane graph, or run eagerly)
static int enqueue_lane(defer_stage_s* s, int lane_id, cudaStream_t st) {
  if (s->has_prod)
    DEFER_TRY(launch_wait_flag(s->ready_flag(lane_id), s->counter(CTR_WAIT_READY, lane_id), 0, s->status_ptr(),
                               s->timeout_ns, st));
  for (int oi = 0; oi < (int)s->ops.size(); ++oi) {
    const int g = s->op_group.empty() ? -1 : s->op_group[oi];
    if (g >= 0 && oi != s->groups[g].first) continue;          // executed by its group's launch
    const int span_last = g >= 0 ? s->groups[g].last : oi;
    if (s->has_cons && s->hop != HOP_COPY && s->output_writer >= oi && s->output_writer <= span_last)
      DEFER_TRY(launch_wait_flag(s->free_flag(lane_id), s->counter(CTR_WAIT_FREE, lane_id), 1, s->status_ptr(),
                                 s->timeout_ns, st));
    if (g >= 0) {
      DEFER_TRY(launch_conv_mega(s->ops[oi].umma.nplanes, s->groups[g].dev_ops[lane_id], span_last - oi + 1, st));
    } else {
      DEFER_TRY(launch_op(s, lane_id, oi, st));
    }
    if (s->has_prod && s->last_input_reader >= oi && s->last_input_reader <= span_last) {
      uint32_t* remote = reinterpret_cast<uint32_t*>(s->prod_arena + OFF_FREE + lane_id * FLAG_STRIDE);
      DEFER_TRY(launch_signal_flag(remote, s->counter(CTR_SIG_FREE, lane_id), s->status_ptr(), st));
    }
  }
  if (s->has_cons && s->hop == HOP_COPY) {
    // the hop: back-pressure (slot free?) is only checked now, after all compute of this microbatch; the payload goes
    // out through the copy engine as one device-to-device copy over NVLink
    Lane& L = s->lanes[lane_id];
    DEFER_TRY(launch_wait_flag(s->free_flag(lane_id), s->counter(CTR_WAIT_FREE, lane_id), 1, s->status_ptr(), s->timeout_ns, st));
    DEFER_CUDA(cudaMemcpyAsync(L.peer_out, L.buf[s->cfg.output_buf], s->bufs[s->cfg.output_buf].bytes, cudaMemcpyDeviceToDevice, st));
  }
  if (s->has_cons) {
    uint32_t* remote = reinterpret_cast<uint32_t*>(s->cons_arena + OFF_READY + lane_id * FLAG_STRIDE);
    DEFER_TRY(launch_signal_flag(remote, s->counter(CTR_SIG_READY, lane_id), s->status_ptr(), st));
  }
  if (s->cfg.is_last) {
    Lane& L = s->lanes[lane_id];
    const Buf& bo = s->bufs[s->cfg.output_buf];
    DEFER_CUDA(cudaMemcpyAsync(L.out_host, L.buf[s->cfg.output_buf], bo.elems * 4, cudaMemcpyDeviceToHost, st));
    DEFER_CUDA(cudaMemcpyAsync(L.status_host, s->status_ptr(), sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  return DEFER_OK;
}

static void op_costs(defer_stage_s* s, OpRt& op) {
  const defer_op_desc& d = op.d;
  const int fmt = s->cfg.fmt;
  const double nb = s->cfg.batch;
  const Buf& bi = s->bufs[d.in0];
  const Buf& bo = s->bufs[d.out];
  auto ab = [&](const Buf& b) { return (double)elem_bytes(b.elem, fmt); };
  double in_b = nb * bi.h * bi.w * bi.c * ab(bi), out_b = nb * bo.h * bo.w * bo.c * ab(bo);
  switch (d.kind) {
    case DEFER_OP_CONV: {
      double wbytes = (op.backend == 2 || op.backend == 4) ? (double)fmt_bytes_per_elem(fmt) : 4.0;
      // a 1x1 convolution with stride > 1 only ever touches the sampled pixels: count those, not the whole input
      if (d.kh == 1 && d.kw == 1 && (d.sh > 1 || d.sw > 1)) in_b = nb * bo.h * bo.w * bi.c * ab(bi);
      op.alg_bytes = in_b + out_b + ((d.flags & DEFER_FLAG_RESIDUAL) ? out_b : 0.0) +
                     (double)d.kh * d.kw * bi.c * bo.c * wbytes + 2.0 * bo.c * 4.0;
      op.alg_flops = 2.0 * nb * bo.h * bo.w * bo.c * d.kh * d.kw * bi.c;
      break;
    }
    case DEFER_OP_DENSE: {
      double F = (double)bi.h * bi.w * bi.c;
      double wb = s->d_weights_bf16[d.w_kernel] ? 2.0 : 4.0;
      op.alg_bytes = in_b + out_b + F * bo.c * wb + bo.c * 4.0;
      op.alg_flops = 2.0 * nb * F * bo.c;
      op.n_kernels = (bo.c % 4 == 0 && (getenv("DEFER_DENSE_FUSED") == nullptr || atoi(getenv("DEFER_DENSE_FUSED")) != 0)) ? 1 : 2;   // fused: one launch
      break;
    }
    case DEFER_OP_ADD:
      op.alg_bytes = 2 * in_b + out_b;
      op.alg_flops = nb * bi.h * bi.w * bi.c;
      break;
    case DEFER_OP_RESIZE:   // + the two int32 tables
      if (d.mode == DEFER_RESIZE_SAMPLE_W || d.mode == DEFER_RESIZE_SAMPLE_H) {   // an upper bound: every sample at the
                                                                                 // slot's size, its header and its axis' tables
        const int out_len = d.mode == DEFER_RESIZE_SAMPLE_W ? bo.w : bo.h;
        op.alg_bytes = in_b + out_b + nb * (2.0 + out_len * (2.0 + d.kw)) * 4.0;
        op.alg_flops = 2.0 * nb * bo.h * bo.w * bo.c * d.kw;
        break;
      }
      op.alg_bytes = in_b + out_b + (double)s->weight_bytes[d.w_scale] + (double)s->weight_bytes[d.w_kernel];
      op.alg_flops = 2.0 * nb * bo.h * bo.w * bo.c * d.kw;
      break;
    case DEFER_OP_JPEG_DECODE: {   // an upper bound: compressed slot + int16 coefficients + planes + image, at the slot's size
      const double blocks_cap = 3.0 * ((bi.h + 15) / 16 * 2) * ((bi.w + 15) / 16 * 2);
      op.alg_bytes = in_b + nb * blocks_cap * (128.0 + 64.0) + out_b;
      op.alg_flops = 0;
      break;
    }
    case DEFER_OP_PNG_DECODE:   // an upper bound: the slot read, gathered and read again, the scanlines written and
                                // unfiltered at the slot's size, and the image
      op.alg_bytes = 3.0 * (double)bi.bytes + 3.0 * nb * bi.h * (1.0 + 8.0 * bi.w) + out_b;
      op.alg_flops = 0;
      break;
    case DEFER_OP_IMAGE_DECODE: {   // an upper bound: every sample as the larger of a JPEG and a PNG of the slot's size
      const double blocks_cap = 3.0 * ((bi.h + 15) / 16 * 2) * ((bi.w + 15) / 16 * 2);
      op.alg_bytes = 3.0 * (double)bi.bytes + nb * std::max(blocks_cap * (128.0 + 64.0), 3.0 * bi.h * (1.0 + 8.0 * bi.w)) + out_b;
      op.alg_flops = 0;
      break;
    }
    default:
      op.alg_bytes = in_b + out_b;
      op.alg_flops = 0;
  }
}

}  // namespace defer

// =============================================================================================== C-ABI
extern "C" {

const char* defer_last_error(void) { return get_error(); }
int defer_abi_version(void) { return DEFER_ABI_VERSION; }

int defer_device_count(int* count) {
  DEFER_CHECK(count, "defer_device_count: null");
  DEFER_CUDA(cudaGetDeviceCount(count));
  return DEFER_OK;
}

int defer_device_info(int device, char* name, int name_len, int* sm_count, int* cc, uint64_t* hbm_bytes) {
  cudaDeviceProp p;
  DEFER_CUDA(cudaGetDeviceProperties(&p, device));
  if (name && name_len > 0) {
    strncpy(name, p.name, name_len - 1);
    name[name_len - 1] = 0;
  }
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc) *cc = p.major * 10 + p.minor;
  if (hbm_bytes) *hbm_bytes = p.totalGlobalMem;
  return DEFER_OK;
}

int defer_stage_create(const defer_stage_config* cfg, const defer_buf_desc* bufs, int n_bufs, const defer_op_desc* ops,
                       int n_ops, const void* const* weight_ptrs, const uint64_t* weight_nbytes, int n_weights,
                       defer_stage_t* out) {
  DEFER_CHECK(cfg && bufs && ops && out, "defer_stage_create: null argument");
  DEFER_CHECK(cfg->abi_version == DEFER_ABI_VERSION, "ABI version mismatch: caller %d, library %d", cfg->abi_version,
              DEFER_ABI_VERSION);
  DEFER_CHECK(cfg->fmt >= 0 && cfg->fmt <= 2, "bad fmt %d", cfg->fmt);
  DEFER_CHECK(cfg->batch >= 1 && cfg->batch <= 4096, "bad batch %d", cfg->batch);
  DEFER_CHECK(cfg->depth >= 1 && cfg->depth <= MAX_DEPTH, "depth %d out of [1,%d]", cfg->depth, MAX_DEPTH);
  DEFER_CHECK(n_bufs >= 2 && n_ops >= 1, "empty plan (%d buffers, %d ops)", n_bufs, n_ops);
  DEFER_CHECK(cfg->input_buf >= 0 && cfg->input_buf < n_bufs && cfg->output_buf >= 0 && cfg->output_buf < n_bufs &&
                  cfg->input_buf != cfg->output_buf,
              "bad input/output buffer ids");
  DEFER_CHECK(!(cfg->conv_backend == 2 && cfg->fmt == DEFER_FMT_F32), "wgmma conv backend needs BF16X2 or BF16 format");
  int ndev = 0;
  DEFER_CUDA(cudaGetDeviceCount(&ndev));
  DEFER_CHECK(cfg->device >= 0 && cfg->device < ndev, "device %d not present (%d visible)", cfg->device, ndev);
  {
    cudaDeviceProp prop;
    DEFER_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    DEFER_CHECK(prop.major == 9, "device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major,
                prop.minor);
  }

  defer_stage_s* s = new defer_stage_s();
  s->cfg = *cfg;
  {
    const char* hm = getenv("DEFER_HOP");
    s->hop = HOP_COPY;
    if (hm && !strcmp(hm, "tma")) s->hop = HOP_TMA;
    else if (hm && !strcmp(hm, "direct")) s->hop = HOP_DIRECT;
  }
  if (cfg->wait_timeout_ms > 0) s->timeout_ns = (unsigned long long)cfg->wait_timeout_ms * 1000000ull;
  int rc = DEFER_OK;
  auto fail = [&](int code) {
    defer_stage_destroy(s);
    return code;
  };
  if ((rc = set_device(s)) != DEFER_OK) return fail(rc);

  // ---- buffers
  for (int i = 0; i < n_bufs; ++i) {
    Buf b;
    b.h = bufs[i].h; b.w = bufs[i].w; b.c = bufs[i].c; b.elem = bufs[i].elem;
    if (b.h < 1 || b.w < 1 || b.c < 1 ||
        (b.elem != DEFER_BUF_ACT && b.elem != DEFER_BUF_F32 && b.elem != DEFER_BUF_U8 && b.elem != DEFER_BUF_JPEG &&
         b.elem != DEFER_BUF_PNG && b.elem != DEFER_BUF_IMAGE)) {
      set_error("buffer %d: bad descriptor (%d,%d,%d,elem %d)", i, b.h, b.w, b.c, b.elem);
      return fail(DEFER_ERR_INVALID);
    }
    if (b.elem == DEFER_BUF_U8) {   // the first stage's image, or that image resized
      bool resized = false;
      for (int j = 0; j < n_ops; ++j)
        resized |= ops[j].out == i && (ops[j].kind == DEFER_OP_RESIZE || ops[j].kind == DEFER_OP_JPEG_DECODE ||
                                       ops[j].kind == DEFER_OP_PNG_DECODE || ops[j].kind == DEFER_OP_IMAGE_DECODE);
      if (!cfg->is_first || (i != cfg->input_buf && !resized)) {
        set_error("buffer %d: a U8 buffer is legal only as the first stage's input buffer or the output of a RESIZE, "
                  "JPEG_DECODE, PNG_DECODE or IMAGE_DECODE op", i);
        return fail(DEFER_ERR_INVALID);
      }
    }
    if (b.elem == DEFER_BUF_JPEG && (!cfg->is_first || i != cfg->input_buf || b.c != 3 ||
                                     !jpeg_bound_ok(b.h, b.w))) {
      set_error("buffer %d: a JPEG buffer is legal only as the first stage's input buffer, (H, W, 3) with "
                "H * W * 24 + %d < 2^31", i, DEFER_JPEG_SUBSEQ_BITS);
      return fail(DEFER_ERR_INVALID);
    }
    if (b.elem == DEFER_BUF_PNG && (!cfg->is_first || i != cfg->input_buf || b.c != 3 || !png_bound_ok(b.h, b.w))) {
      set_error("buffer %d: a PNG buffer is legal only as the first stage's input buffer, (H, W, 3) with "
                "DEFER_PNG_SLOT_BYTES(H, W) < 2^31", i);
      return fail(DEFER_ERR_INVALID);
    }
    if (b.elem == DEFER_BUF_IMAGE && (!cfg->is_first || i != cfg->input_buf || b.c != 3 || !image_bound_ok(b.h, b.w))) {
      set_error("buffer %d: an image buffer is legal only as the first stage's input buffer, (H, W, 3) with "
                "H * W * 24 + %d < 2^31 and DEFER_PNG_SLOT_BYTES(H, W) < 2^31", i, DEFER_JPEG_SUBSEQ_BITS);
      return fail(DEFER_ERR_INVALID);
    }
    b.elems = (size_t)cfg->batch * b.h * b.w * b.c;
    b.bytes = b.elem == DEFER_BUF_PNG || b.elem == DEFER_BUF_IMAGE
                  ? (size_t)cfg->batch * DEFER_PNG_SLOT_BYTES((size_t)b.h, (size_t)b.w)
                  : buf_bytes(b, cfg->fmt);
    s->bufs.push_back(b);
  }
  if (cfg->is_first && s->bufs[cfg->input_buf].elem == DEFER_BUF_ACT) {
    set_error("first stage input must be an F32 or U8 buffer");
    return fail(DEFER_ERR_INVALID);
  }
  if (cfg->is_last && s->bufs[cfg->output_buf].elem != DEFER_BUF_F32) {
    set_error("last stage output must be an F32 buffer");
    return fail(DEFER_ERR_INVALID);
  }

  // ---- weights (fp32 copies; the caller keeps its host arrays, cf. src/node.py:34)
  s->d_weights.assign(n_weights, nullptr);
  s->d_weights_bf16.assign(n_weights, nullptr);
  s->weight_bytes.assign(n_weights, 0);
  for (int i = 0; i < n_weights; ++i) {
    size_t nbytes = weight_nbytes[i];
    if (!weight_ptrs[i] || nbytes == 0 || nbytes % 4) {
      set_error("weight %d: null or bad size %zu", i, nbytes);
      return fail(DEFER_ERR_INVALID);
    }
    void* d = nullptr;
    if (cudaMalloc(&d, nbytes) != cudaSuccess) {
      set_error("cudaMalloc(%zu) for weight %d failed", nbytes, i);
      return fail(DEFER_ERR_CUDA);
    }
    s->d_weights[i] = d;
    s->weight_bytes[i] = nbytes;
    if (cudaMemcpy(d, weight_ptrs[i], nbytes, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("H2D copy of weight %d failed", i);
      return fail(DEFER_ERR_CUDA);
    }
  }

  // ---- ops: validate, pick backends
  std::vector<int> writer(n_bufs, -1);
  for (int i = 0; i < n_ops; ++i) {
    OpRt op;
    op.d = ops[i];
    const defer_op_desc& d = op.d;
    auto okbuf = [&](int id) { return id >= 0 && id < n_bufs; };
    if (!okbuf(d.in0) || !okbuf(d.out) || (d.in1 >= 0 && !okbuf(d.in1))) {
      set_error("op %d: bad buffer ids (%d,%d,%d)", i, d.in0, d.in1, d.out);
      return fail(DEFER_ERR_INVALID);
    }
    if (writer[d.out] >= 0 || d.out == cfg->input_buf) {
      set_error("op %d: buffer %d written twice (plan must be SSA)", i, d.out);
      return fail(DEFER_ERR_INVALID);
    }
    if ((d.in0 != cfg->input_buf && writer[d.in0] < 0) || (d.in1 >= 0 && d.in1 != cfg->input_buf && writer[d.in1] < 0)) {
      set_error("op %d reads a buffer that no earlier op wrote", i);
      return fail(DEFER_ERR_INVALID);
    }
    writer[d.out] = i;
    auto okw = [&](int id) { return id >= -1 && id < n_weights; };
    if (!okw(d.w_kernel) || !okw(d.w_scale) || !okw(d.w_shift)) {
      set_error("op %d: bad weight ids", i);
      return fail(DEFER_ERR_INVALID);
    }
    const Buf& bi = s->bufs[d.in0];
    const Buf& bo = s->bufs[d.out];
    if ((bi.elem == DEFER_BUF_U8 && d.kind != DEFER_OP_PREPROCESS && d.kind != DEFER_OP_RESIZE) ||
        (d.in1 >= 0 && s->bufs[d.in1].elem == DEFER_BUF_U8)) {
      set_error("op %d: only a RESIZE or PREPROCESS op may read a U8 buffer (as in0)", i);
      return fail(DEFER_ERR_INVALID);
    }
    if ((bi.elem == DEFER_BUF_JPEG) != (d.kind == DEFER_OP_JPEG_DECODE) || (d.in1 >= 0 && s->bufs[d.in1].elem == DEFER_BUF_JPEG)) {
      set_error("op %d: a JPEG buffer is read only by a JPEG_DECODE op (as in0), which reads nothing else", i);
      return fail(DEFER_ERR_INVALID);
    }
    if ((bi.elem == DEFER_BUF_PNG) != (d.kind == DEFER_OP_PNG_DECODE) || (d.in1 >= 0 && s->bufs[d.in1].elem == DEFER_BUF_PNG)) {
      set_error("op %d: a PNG buffer is read only by a PNG_DECODE op (as in0), which reads nothing else", i);
      return fail(DEFER_ERR_INVALID);
    }
    if ((bi.elem == DEFER_BUF_IMAGE) != (d.kind == DEFER_OP_IMAGE_DECODE) ||
        (d.in1 >= 0 && s->bufs[d.in1].elem == DEFER_BUF_IMAGE)) {
      set_error("op %d: an image buffer is read only by an IMAGE_DECODE op (as in0), which reads nothing else", i);
      return fail(DEFER_ERR_INVALID);
    }
    if (d.kind != DEFER_OP_PREPROCESS && d.kind != DEFER_OP_RESIZE && d.mode != 0) {
      set_error("op %d: mode %d is meaningful only on a PREPROCESS or RESIZE op and must be 0 here", i, d.mode);
      return fail(DEFER_ERR_INVALID);
    }
    switch (d.kind) {
      case DEFER_OP_CONV: {
        int ho = (bi.h + d.pad_t + d.pad_b - d.kh) / d.sh + 1, wo = (bi.w + d.pad_l + d.pad_r - d.kw) / d.sw + 1;
        if (d.kh < 1 || d.kw < 1 || d.sh < 1 || d.sw < 1 || ho != bo.h || wo != bo.w || d.w_kernel < 0 ||
            s->weight_bytes[d.w_kernel] != (size_t)d.kh * d.kw * bi.c * bo.c * 4 || bo.elem != DEFER_BUF_ACT) {
          set_error("op %d (conv): inconsistent shapes in=(%d,%d,%d) out=(%d,%d,%d) k=%dx%d s=%dx%d", i, bi.h, bi.w, bi.c,
                    bo.h, bo.w, bo.c, d.kh, d.kw, d.sh, d.sw);
          return fail(DEFER_ERR_INVALID);
        }
        if ((d.flags & DEFER_FLAG_RESIDUAL) && (d.in1 < 0 || s->bufs[d.in1].elems != bo.elems)) {
          set_error("op %d (conv): residual buffer missing or wrong size", i);
          return fail(DEFER_ERR_INVALID);
        }
        bool can_umma = cfg->fmt != DEFER_FMT_F32 && bi.elem == DEFER_BUF_ACT &&
                        umma_conv_supported(cfg->fmt, cfg->batch, bi.h, bi.w, bi.c, bo.h, bo.w, bo.c, d.kh, d.kw, d.sh, d.sw,
                                            d.pad_t, d.pad_l);
        if (cfg->conv_backend == 1) can_umma = false;
        op.backend = can_umma ? 2 : 1;
        op.kname = can_umma ? "conv_umma_kernel" : "conv_simt_kernel";
        // RGB stem (fp32 image in, few input channels): im2col to a K_pad-channel patch matrix, then the wgmma kernel
        // as a 1x1 conv (the fp32 FFMA stem runs 147 MACs per output on the SIMT pipe; the tensor cores take them instead)
        // DEFER_TC_STEM: 0 off, 1 strided stems only (ResNet 7x7/2), 2 (default) every eligible first conv (VGG's 3x3/1 too)
        const int tc_stem = getenv("DEFER_TC_STEM") ? atoi(getenv("DEFER_TC_STEM")) : 2;
        const int K = d.kh * d.kw * bi.c;
        if (tc_stem && cfg->conv_backend != 1 && cfg->fmt != DEFER_FMT_F32 && bi.elem == DEFER_BUF_F32 && bi.c < 64 && K <= 256 &&
            bo.c % 64 == 0 && !(d.flags & DEFER_FLAG_RESIDUAL) && d.sh <= 2 && d.sw <= 2 &&
            (tc_stem >= 2 || (d.sh == 2 && d.sw == 2))) {
          op.backend = 4;
          op.k_pad = (K + 63) / 64 * 64;
          op.kname = "stem_im2col+conv_umma_kernel";
          op.n_kernels = 2;
        }
        break;
      }
      case DEFER_OP_MAXPOOL:
        op.kname = "maxpool_kernel";
        if (bi.c != bo.c || bi.elem != DEFER_BUF_ACT || bo.elem != DEFER_BUF_ACT) {
          set_error("op %d (maxpool): bad buffers", i);
          return fail(DEFER_ERR_INVALID);
        }
        break;
      case DEFER_OP_GAP: op.kname = "gap_kernel"; break;
      case DEFER_OP_DENSE: {
        op.kname = (bo.c % 4 == 0 && (getenv("DEFER_DENSE_FUSED") == nullptr || atoi(getenv("DEFER_DENSE_FUSED")) != 0)) ? "dense_fused_kernel" : "dense_partial_kernel";
        size_t F = (size_t)bi.h * bi.w * bi.c;
        if (d.w_kernel < 0 || s->weight_bytes[d.w_kernel] != F * bo.c * 4 || bi.elem != DEFER_BUF_ACT) {
          set_error("op %d (dense): kernel size mismatch (F=%zu U=%d)", i, F, bo.c);
          return fail(DEFER_ERR_INVALID);
        }
        size_t need = dense_workspace_bytes(cfg->batch, (int)F, bo.c);
        if (need > s->max_dense_partial) s->max_dense_partial = need;
        if (cfg->fmt == DEFER_FMT_BF16 && !s->d_weights_bf16[d.w_kernel]) {
          void* wb = nullptr;
          if (cudaMalloc(&wb, F * bo.c * 2) != cudaSuccess) {
            set_error("cudaMalloc bf16 dense kernel failed");
            return fail(DEFER_ERR_CUDA);
          }
          s->d_weights_bf16[d.w_kernel] = wb;
          if ((rc = launch_f32_to_bf16((const float*)s->d_weights[d.w_kernel], wb, F * bo.c, 0)) != DEFER_OK) return fail(rc);
        }
        break;
      }
      case DEFER_OP_SOFTMAX:
        op.kname = "softmax_kernel";
        if (bi.elem != DEFER_BUF_F32 || bo.elem != DEFER_BUF_F32) {
          set_error("op %d (softmax): needs F32 buffers", i);
          return fail(DEFER_ERR_INVALID);
        }
        break;
      case DEFER_OP_AFFINE:
      case DEFER_OP_RELU:
      case DEFER_OP_ADD:
        op.kname = "eltwise_kernel";
        if (bi.elem != DEFER_BUF_ACT || bo.elem != DEFER_BUF_ACT || bi.elems != bo.elems ||
            (d.kind == DEFER_OP_ADD && (d.in1 < 0 || s->bufs[d.in1].elems != bi.elems))) {
          set_error("op %d (eltwise): bad buffers", i);
          return fail(DEFER_ERR_INVALID);
        }
        break;
      case DEFER_OP_PAD: op.kname = "pad_kernel"; break;
      case DEFER_OP_COPY:
        op.kname = "copy_kernel";
        if (bi.elems != bo.elems) {
          set_error("op %d (copy): size mismatch", i);
          return fail(DEFER_ERR_INVALID);
        }
        break;
      case DEFER_OP_PREPROCESS:
        if (d.mode != DEFER_PRE_CAFFE && d.mode != DEFER_PRE_TF) {
          set_error("op %d (preprocess): unknown mode %d (caffe %d, tf %d)", i, d.mode, DEFER_PRE_CAFFE, DEFER_PRE_TF);
          return fail(DEFER_ERR_INVALID);
        }
        op.kname = d.mode == DEFER_PRE_TF ? "preprocess_tf_kernel" : "preprocess_kernel";
        if (bi.elem != DEFER_BUF_U8 || bi.c != 3) {
          set_error("op %d (preprocess): input must be a U8 buffer with 3 channels (elem %d, c %d)", i, bi.elem, bi.c);
          return fail(DEFER_ERR_INVALID);
        }
        if (bo.elem != DEFER_BUF_F32 || bo.h != bi.h || bo.w != bi.w || bo.c != bi.c) {
          set_error("op %d (preprocess): output must be an F32 buffer of the input's shape", i);
          return fail(DEFER_ERR_INVALID);
        }
        if (d.mode == DEFER_PRE_TF) {   // Keras hard-codes 127.5 and 1: nothing to upload
          if (d.w_kernel >= 0 || d.w_scale >= 0 || d.w_shift >= 0) {
            set_error("op %d (preprocess, tf): takes no weights (w_kernel %d, w_scale %d, w_shift %d)", i, d.w_kernel,
                      d.w_scale, d.w_shift);
            return fail(DEFER_ERR_INVALID);
          }
          break;
        }
        if (d.w_shift < 0 || s->weight_bytes[d.w_shift] != 3 * sizeof(float)) {
          set_error("op %d (preprocess): w_shift must hold 3 fp32 values", i);
          return fail(DEFER_ERR_INVALID);
        }
        memcpy(op.pre_shift, weight_ptrs[d.w_shift], sizeof op.pre_shift);
        break;
      case DEFER_OP_RESIZE: {
        op.kname = "resize_u8_kernel";
        if (bi.elem != DEFER_BUF_U8 || bo.elem != DEFER_BUF_U8 || bi.c != 3 || bo.c != 3) {
          set_error("op %d (resize): needs U8 buffers with 3 channels (in elem %d c %d, out elem %d c %d)", i, bi.elem, bi.c,
                    bo.elem, bo.c);
          return fail(DEFER_ERR_INVALID);
        }
        if (d.mode == DEFER_RESIZE_SAMPLE_W || d.mode == DEFER_RESIZE_SAMPLE_H) {   // images of mixed sizes
          const bool horiz = d.mode == DEFER_RESIZE_SAMPLE_W;
          op.kname = "resize_frames_u8_kernel";
          auto& f = s->frames;
          if (d.in1 >= 0 || d.flags || d.w_kernel >= 0 || d.w_scale >= 0 || d.w_shift >= 0) {
            set_error("op %d (resize, per sample): takes no weights, in1 or flags (its tables come with each microbatch)", i);
            return fail(DEFER_ERR_INVALID);
          }
          const bool from_input = d.in0 == cfg->input_buf || (s->dec.op >= 0 && d.in0 == ops[s->dec.op].out);
          if (horiz ? (!from_input || bo.h != bi.h || f.op_w >= 0) : (bo.w != bi.w || f.op_h >= 0)) {
            set_error("op %d (resize, per sample): SAMPLE_W maps the stage input (H, W) to (H, W_out), SAMPLE_H maps (H, W_out) "
                      "to (H_out, W_out), one of each per stage (got %dx%d -> %dx%d, mode %d)", i, bi.h, bi.w, bo.h, bo.w, d.mode);
            return fail(DEFER_ERR_INVALID);
          }
          // kw holds the axis' taps for every source length up to the bound: at most the widest filter's (lanczos, support 3)
          const int in_len = horiz ? bi.w : bi.h, out_len = horiz ? bo.w : bo.h;
          const int kmax = 2 * (int)ceil(3.0 * fmax((double)in_len / out_len, 1.0)) + 1;
          if (d.kw < 1 || d.kw > kmax) {
            set_error("op %d (resize, per sample): kw = %d taps, needs 1 <= kw <= %d for %d -> %d", i, d.kw, kmax, in_len, out_len);
            return fail(DEFER_ERR_INVALID);
          }
          if (horiz) {
            f.op_w = i;
            f.H = bi.h; f.W = bi.w; f.W_out = bo.w; f.kw_w = d.kw;
          } else {
            f.op_h = i;
            f.H_out = bo.h; f.kw_h = d.kw;
          }
          break;
        }
        if (d.mode != 0 && d.mode != DEFER_RESIZE_W && d.mode != DEFER_RESIZE_H) {
          set_error("op %d (resize): unknown mode %d (0, SAMPLE_W %d, SAMPLE_H %d, W %d, H %d)", i, d.mode,
                    DEFER_RESIZE_SAMPLE_W, DEFER_RESIZE_SAMPLE_H, DEFER_RESIZE_W, DEFER_RESIZE_H);
          return fail(DEFER_ERR_INVALID);
        }
        if (d.in1 >= 0 || d.flags || d.w_shift >= 0 ||
            (d.mode == 0 ? (bi.h != bo.h) == (bi.w != bo.w) : d.mode == DEFER_RESIZE_W ? bi.h != bo.h : bi.w != bo.w)) {
          set_error("op %d (resize): mode 0 needs exactly one axis to change, mode W / H only its axis (%dx%d -> %dx%d, mode "
                    "%d), no in1 / flags / w_shift", i, bi.h, bi.w, bo.h, bo.w, d.mode);
          return fail(DEFER_ERR_INVALID);
        }
        const bool horiz = resize_horizontal(d, bi, bo);
        const int in_len = horiz ? bi.w : bi.h, out_len = horiz ? bo.w : bo.h, ksize = d.kw;
        if (ksize < 1 || d.w_scale < 0 || d.w_kernel < 0 || s->weight_bytes[d.w_scale] != (size_t)out_len * 2 * 4 ||
            s->weight_bytes[d.w_kernel] != (size_t)out_len * ksize * 4) {
          set_error("op %d (resize): w_scale must hold int32 [%d, 2] (first, count) and w_kernel int32 [%d, kw = %d] taps", i,
                    out_len, out_len, ksize);
          return fail(DEFER_ERR_INVALID);
        }
        const int32_t* b = static_cast<const int32_t*>(weight_ptrs[d.w_scale]);
        for (int o = 0; o < out_len; ++o) {
          const int first = b[2 * o], count = b[2 * o + 1];
          if (first < 0 || count < 1 || count > ksize || first > in_len - count) {
            set_error("op %d (resize): output %d reads source [%d, %d + %d); needs 0 <= first, 1 <= count <= kw = %d, "
                      "first + count <= %d", i, o, first, first, count, ksize, in_len);
            return fail(DEFER_ERR_INVALID);
          }
        }
        break;
      }
      case DEFER_OP_JPEG_DECODE:
        op.kname = "jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel";
        op.n_kernels = 3;
        if (d.in0 != cfg->input_buf || bo.elem != DEFER_BUF_U8 || bo.h != bi.h || bo.w != bi.w || bo.c != 3 || d.in1 >= 0 ||
            d.flags || d.mode || d.w_kernel >= 0 || d.w_scale >= 0 || d.w_shift >= 0 || s->dec.op >= 0) {
          set_error("op %d (jpeg decode): maps the stage's JPEG input (H, W, 3) to a U8 (H, W, 3) buffer, once, with no weights, "
                    "in1, flags or mode", i);
          return fail(DEFER_ERR_INVALID);
        }
        s->dec.op = i;
        s->dec.kind = d.kind;
        s->dec.block_ints = DEFER_JPEG_BLOCK_INTS;
        break;
      case DEFER_OP_PNG_DECODE:
        op.kname = "png_inflate_kernel+png_unfilter_kernel+png_expand_kernel";
        op.n_kernels = 3;
        if (d.in0 != cfg->input_buf || bo.elem != DEFER_BUF_U8 || bo.h != bi.h || bo.w != bi.w || bo.c != 3 || d.in1 >= 0 ||
            d.flags || d.mode || d.w_kernel >= 0 || d.w_scale >= 0 || d.w_shift >= 0 || s->dec.op >= 0) {
          set_error("op %d (png decode): maps the stage's PNG input (H, W, 3) to a U8 (H, W, 3) buffer, once, with no weights, "
                    "in1, flags or mode (and no other decode op)", i);
          return fail(DEFER_ERR_INVALID);
        }
        s->dec.op = i;
        s->dec.kind = d.kind;
        s->dec.block_ints = DEFER_PNG_BLOCK_INTS;
        break;
      case DEFER_OP_IMAGE_DECODE:
        op.kname = "jpeg_entropy_kernel+jpeg_idct_kernel+jpeg_color_kernel+png_inflate_kernel+png_unfilter_kernel+"
                   "png_expand_kernel";
        op.n_kernels = 6;
        if (d.in0 != cfg->input_buf || bo.elem != DEFER_BUF_U8 || bo.h != bi.h || bo.w != bi.w || bo.c != 3 || d.in1 >= 0 ||
            d.flags || d.mode || d.w_kernel >= 0 || d.w_scale >= 0 || d.w_shift >= 0 || s->dec.op >= 0) {
          set_error("op %d (image decode): maps the stage's image input (H, W, 3) to a U8 (H, W, 3) buffer, once, with no "
                    "weights, in1, flags or mode (and no other decode op)", i);
          return fail(DEFER_ERR_INVALID);
        }
        s->dec.op = i;
        s->dec.kind = d.kind;
        s->dec.block_ints = DEFER_IMAGE_BLOCK_INTS;
        break;
      default:
        set_error("op %d: unknown kind %d", i, d.kind);
        return fail(DEFER_ERR_INVALID);
    }
    s->ops.push_back(op);
  }
  if (writer[cfg->output_buf] < 0) {
    set_error("no op writes the output buffer %d", cfg->output_buf);
    return fail(DEFER_ERR_INVALID);
  }
  s->output_writer = writer[cfg->output_buf];
  if (s->frames.op_w >= 0 || s->frames.op_h >= 0) {
    auto& f = s->frames;
    if (f.op_w < 0 || f.op_h < 0 || ops[f.op_h].in0 != ops[f.op_w].out) {
      set_error("the per-sample resize ops come as a pair: SAMPLE_W on the stage input, SAMPLE_H on its output (ops %d, %d)",
                f.op_w, f.op_h);
      return fail(DEFER_ERR_INVALID);
    }
    f.block_ints = 2 + (size_t)f.W_out * (2 + f.kw_w) + (size_t)f.H_out * (2 + f.kw_h);
  }
  if (s->dec.op >= 0 && (s->frames.op_w < 0 || ops[s->frames.op_w].in0 != ops[s->dec.op].out)) {
    set_error("the %s_DECODE op (op %d) feeds the per-sample resize pair: its output is SAMPLE_W's input",
              s->dec.kind == DEFER_OP_IMAGE_DECODE ? "IMAGE" : dec_name(s, true), s->dec.op);
    return fail(DEFER_ERR_INVALID);
  }
  for (int i = 0; i < n_ops; ++i)
    if (ops[i].in0 == cfg->input_buf || ops[i].in1 == cfg->input_buf) s->last_input_reader = i;
  if (s->last_input_reader < 0) {
    set_error("no op reads the input buffer");
    return fail(DEFER_ERR_INVALID);
  }
  for (auto& op : s->ops) op_costs(s, op);
  // DEFER_FOLD_AFFINE=1: fold each AFFINE op whose input a wgmma conv of this stage writes into that conv (one per conv).
  // The conv keeps its own store only when another op reads that buffer or it is the stage output.  The SIMT / F32 path
  // keeps the standalone op, and so does the RGB stem.  Opt-in: measured on H100 the folded ResNet V2 step is slower
  // (the epilogue's pair-wise stores are less coalesced than eltwise_kernel's float4 pass; BASELINE.md section 4).
  {
    const char* fe = getenv("DEFER_FOLD_AFFINE");
    const bool fold = fe != nullptr && atoi(fe) != 0;
    for (int ai = 0; fold && ai < n_ops; ++ai) {
      OpRt& aff = s->ops[ai];
      const defer_op_desc& d = aff.d;
      if (d.kind != DEFER_OP_AFFINE || d.w_scale < 0 || d.w_shift < 0) continue;
      const int ci = writer[d.in0];
      if (ci < 0 || s->ops[ci].d.kind != DEFER_OP_CONV || s->ops[ci].backend != 2 || s->ops[ci].aff_op >= 0) continue;
      OpRt& conv = s->ops[ci];
      bool needed = d.in0 == cfg->output_buf;
      for (int oi = 0; oi < n_ops; ++oi)
        if (oi != ai && (ops[oi].in0 == d.in0 || ops[oi].in1 == d.in0)) needed = true;
      aff.folded_into = ci;
      aff.n_kernels = 0;
      conv.aff_op = ai;
      conv.store_out = needed;
      conv.kname = "conv_umma_aff_kernel";
      aff.kname = "affine (fused into " + conv.kname + ")";
      conv.alg_bytes += aff.alg_bytes / 2;     // + the affine op's output (op_costs counted its input and output)
      if (!needed) conv.alg_bytes -= aff.alg_bytes / 2;
      aff.alg_bytes = 0;
      if (s->output_writer == ai) s->output_writer = ci;   // HOP_TMA / HOP_DIRECT: wait for the slot before the conv
    }
  }

  // ---- arena: ctrl + input slots (exported to the upstream stage)
  size_t in_bytes = s->bufs[cfg->input_buf].bytes;
  s->slot_stride = (in_bytes + 1023) / 1024 * 1024;
  if (s->frames.op_w >= 0) {   // the lane's table blocks follow its input slot (zeroed with the arena below)
    s->frames.tables_off = s->slot_stride;
    s->slot_stride += ((size_t)cfg->batch * s->frames.block_ints * 4 + 1023) / 1024 * 1024;
  }
  if (s->dec.op >= 0) {       // then the JPEG or PNG blocks (zeroed with the arena too)
    const Buf& bi = s->bufs[cfg->input_buf];
    s->dec.blocks_off = s->slot_stride;
    s->slot_stride += ((size_t)cfg->batch * s->dec.block_ints * 4 + 1023) / 1024 * 1024;
    s->dec.ws_bytes = s->dec.kind == DEFER_OP_PNG_DECODE     ? png_workspace_bytes(bi.h, bi.w, cfg->batch)
                      : s->dec.kind == DEFER_OP_IMAGE_DECODE ? image_workspace_bytes(bi.h, bi.w, cfg->batch)
                                                             : jpeg_workspace_bytes(bi.h, bi.w, cfg->batch);
  }
  s->arena_bytes = CTRL_BYTES + s->slot_stride * cfg->depth;
  if (cudaMalloc((void**)&s->arena, s->arena_bytes) != cudaSuccess) {
    set_error("cudaMalloc arena (%zu bytes) failed", s->arena_bytes);
    return fail(DEFER_ERR_CUDA);
  }
  if (cudaMemset(s->arena, 0, s->arena_bytes) != cudaSuccess) {
    set_error("cudaMemset arena failed");
    return fail(DEFER_ERR_CUDA);
  }

  // ---- lanes
  s->lanes.resize(cfg->depth);
  for (int l = 0; l < cfg->depth; ++l) {
    Lane& L = s->lanes[l];
    if (cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&L.done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&L.join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreate(&L.t0) != cudaSuccess || cudaEventCreate(&L.t1) != cudaSuccess) {
      set_error("stream/event creation failed");
      return fail(DEFER_ERR_CUDA);
    }
    L.buf.assign(n_bufs, nullptr);
    L.buf[cfg->input_buf] = s->arena + CTRL_BYTES + s->slot_stride * l;
    if (s->frames.op_w >= 0) L.tables = reinterpret_cast<int32_t*>(s->arena + CTRL_BYTES + s->slot_stride * l + s->frames.tables_off);
    if (s->dec.op >= 0) {
      L.dec_blocks = reinterpret_cast<int32_t*>(s->arena + CTRL_BYTES + s->slot_stride * l + s->dec.blocks_off);
      if (cudaMalloc(&L.dec_ws, s->dec.ws_bytes) != cudaSuccess) {
        set_error("cudaMalloc %s decode workspace (%zu bytes) failed", dec_name(s, true), s->dec.ws_bytes);
        return fail(DEFER_ERR_CUDA);
      }
      s->workspace.push_back(L.dec_ws);
    }
    for (int b = 0; b < n_bufs; ++b) {
      if (b == cfg->input_buf) continue;
      if (b == cfg->output_buf && !cfg->is_last && s->hop != HOP_COPY) continue;  // bound to the consumer's slot at link time
      void* p = nullptr;
      size_t bytes = (s->bufs[b].bytes + 255) / 256 * 256;
      if (cudaMalloc(&p, bytes) != cudaSuccess) {
        set_error("cudaMalloc workspace buffer %d (%zu bytes) failed", b, bytes);
        return fail(DEFER_ERR_CUDA);
      }
      s->workspace.push_back(p);
      L.buf[b] = p;
    }
    if (s->max_dense_partial) {
      if (cudaMalloc((void**)&L.dense_partial, s->max_dense_partial) != cudaSuccess) {
        set_error("cudaMalloc dense partial failed");
        return fail(DEFER_ERR_CUDA);
      }
      s->workspace.push_back(L.dense_partial);
      if (cudaMemset(L.dense_partial, 0, s->max_dense_partial) != cudaSuccess) {   // arrival counters of the fused dense kernel
        set_error("cudaMemset dense workspace failed");
        return fail(DEFER_ERR_CUDA);
      }
    }
    if (cfg->is_last) {
      if (cudaMallocHost((void**)&L.out_host, s->bufs[cfg->output_buf].elems * 4) != cudaSuccess ||
          cudaMallocHost((void**)&L.status_host, sizeof(int)) != cudaSuccess) {
        set_error("cudaMallocHost result buffer failed");
        return fail(DEFER_ERR_CUDA);
      }
      *L.status_host = 0;
    }
    L.umma.resize(n_ops);
  }
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("device sync after stage setup failed: %s", cudaGetErrorString(cudaGetLastError()));
    return fail(DEFER_ERR_CUDA);
  }
  *out = s;
  return DEFER_OK;
}

int defer_stage_destroy(defer_stage_t s) {
  if (!s) return DEFER_OK;
  cudaSetDevice(s->cfg.device);
  cudaDeviceSynchronize();
  for (auto& L : s->lanes) {
    if (L.exec) cudaGraphExecDestroy(L.exec);
    if (L.graph) cudaGraphDestroy(L.graph);
    if (L.stream) cudaStreamDestroy(L.stream);
    if (L.done) cudaEventDestroy(L.done);
    if (L.join) cudaEventDestroy(L.join);
    if (L.t0) cudaEventDestroy(L.t0);
    if (L.t1) cudaEventDestroy(L.t1);
    for (auto& ua : L.umma) umma_conv_unbind(&ua);
    if (L.out_host) cudaFreeHost(L.out_host);
    if (L.status_host) cudaFreeHost(L.status_host);
  }
  for (auto& op : s->ops)
    if (op.backend == 2 || op.backend == 4) umma_conv_release(op.umma);
  for (void* p : s->workspace) cudaFree(p);
  for (void* p : s->d_weights) if (p) cudaFree(p);
  for (void* p : s->d_weights_bf16) if (p) cudaFree(p);
  if (s->cons_arena && s->cons_is_ipc) cudaIpcCloseMemHandle(s->cons_arena);
  if (s->prod_arena && s->prod_is_ipc) cudaIpcCloseMemHandle(s->prod_arena);
  for (auto& m : s->marks) if (m.ev) cudaEventDestroy(m.ev);
  if (s->job_t0) cudaEventDestroy(s->job_t0);
  if (s->job_t1) cudaEventDestroy(s->job_t1);
  if (s->flush_buf) cudaFree(s->flush_buf);
  if (s->arena) cudaFree(s->arena);
  delete s;
  return DEFER_OK;
}

int defer_stage_describe(defer_stage_t s, char* buf, size_t buf_len) {
  DEFER_CHECK(s && buf && buf_len > 0, "describe: null");
  std::string o;
  char line[512];
  static const char* fm[] = {"f32", "bf16x2", "bf16"};
  snprintf(line, sizeof line, "stage device=%d fmt=%s batch=%d depth=%d first=%d last=%d ops=%zu prod=%d cons=%d\n",
           s->cfg.device, fm[s->cfg.fmt], s->cfg.batch, s->cfg.depth, s->cfg.is_first, s->cfg.is_last, s->ops.size(),
           (int)s->has_prod, (int)s->has_cons);
  o += line;
  for (size_t i = 0; i < s->ops.size(); ++i) {
    const OpRt& op = s->ops[i];
    const Buf& bi = s->bufs[op.d.in0];
    const Buf& bo = s->bufs[op.d.out];
    if (!s->op_group.empty() && s->op_group[i] >= 0 && (int)i == s->groups[s->op_group[i]].first) {
      snprintf(line, sizeof line, "  -- megakernel group: ops %d..%d in one cluster launch --\n", s->groups[s->op_group[i]].first,
               s->groups[s->op_group[i]].last);
      o += line;
    }
    snprintf(line, sizeof line, "  [%2zu] %-22s in b%-3d(%d,%d,%d) res b%-3d -> b%-3d(%d,%d,%d) k=%dx%d s=%d flags=%u  %.3f MB %.3f GF\n", i,
             op.kname.c_str(), op.d.in0, bi.h, bi.w, bi.c, op.d.in1, op.d.out, bo.h, bo.w, bo.c, op.d.kh, op.d.kw, op.d.sh,
             op.d.flags, op.alg_bytes / 1e6, op.alg_flops / 1e9);
    o += line;
    if ((op.backend == 2 || op.backend == 4) && op.umma.ready) {
      const UmmaConvPlan& u = op.umma;
      snprintf(line, sizeof line, "       wgmma tiles: m=%d x n=%d (BN %d) x k-splits %d%s, %d k-blocks, ring %d -> %d CTAs\n",
               u.m_tiles, u.cout / u.bn, u.bn, u.splits, u.cluster ? " (cluster, DSMEM reduce)" : "",
               u.k_blocks, u.stages, u.m_tiles * (u.cout / u.bn) * u.splits);
      o += line;
    }
  }
  strncpy(buf, o.c_str(), buf_len - 1);
  buf[buf_len - 1] = 0;
  return DEFER_OK;
}

int defer_stage_io_bytes(defer_stage_t s, uint64_t* in_bytes, uint64_t* out_bytes) {
  DEFER_CHECK(s, "io_bytes: null");
  if (in_bytes) *in_bytes = s->bufs[s->cfg.input_buf].bytes;
  if (out_bytes) *out_bytes = s->bufs[s->cfg.output_buf].bytes;
  return DEFER_OK;
}

// ------------------------------------------------------------------------------------------ linking
static int fill_token(defer_stage_t s, int role, LinkToken* t) {
  memset(t, 0, sizeof(*t));
  t->magic = TOKEN_MAGIC;
  t->role = role;
  t->device = s->cfg.device;
  t->pid = (int)getpid();
  t->depth = s->cfg.depth;
  t->fmt = s->cfg.fmt;
  t->batch = s->cfg.batch;
  t->slot_bytes = role == 0 ? s->bufs[s->cfg.input_buf].bytes : s->bufs[s->cfg.output_buf].bytes;
  t->arena_bytes = s->arena_bytes;
  t->off_slots = CTRL_BYTES;
  t->slot_stride = s->slot_stride;
  t->local_base = (uint64_t)(uintptr_t)s->arena;
  return DEFER_OK;
}

static int apply_token(defer_stage_t s, int role, const LinkToken* t, uint8_t* mapped, bool is_ipc) {
  // role == 0: token describes the INPUT side of my consumer -> I become its producer
  // role == 1: token describes the OUTPUT side of my producer -> I become its consumer
  DEFER_CHECK(t->depth == s->cfg.depth && t->fmt == s->cfg.fmt && t->batch == s->cfg.batch,
              "link: depth/fmt/batch mismatch (peer %d/%d/%d, mine %d/%d/%d)", t->depth, t->fmt, t->batch, s->cfg.depth,
              s->cfg.fmt, s->cfg.batch);
  if (role == 0) {
    DEFER_CHECK(!s->cfg.is_last, "link: the last stage has no consumer");
    DEFER_CHECK(t->slot_bytes == s->bufs[s->cfg.output_buf].bytes, "link: my output is %zu bytes, consumer slot is %llu",
                s->bufs[s->cfg.output_buf].bytes, (unsigned long long)t->slot_bytes);
    s->cons_arena = mapped;
    s->cons_is_ipc = is_ipc;
    s->cons_off_slots = t->off_slots;
    s->cons_slot_stride = t->slot_stride;
    for (int l = 0; l < s->cfg.depth; ++l) {
      void* slot = mapped + t->off_slots + t->slot_stride * l;
      if (s->hop == HOP_COPY) s->lanes[l].peer_out = slot;          // output stays local, a copy node ships it
      else s->lanes[l].buf[s->cfg.output_buf] = slot;               // the last op writes the peer slot itself
    }
    s->has_cons = true;
  } else {
    DEFER_CHECK(!s->cfg.is_first, "link: the first stage has no producer");
    DEFER_CHECK(t->slot_bytes == s->bufs[s->cfg.input_buf].bytes, "link: my input is %zu bytes, producer sends %llu",
                s->bufs[s->cfg.input_buf].bytes, (unsigned long long)t->slot_bytes);
    s->prod_arena = mapped;
    s->prod_is_ipc = is_ipc;
    s->has_prod = true;
  }
  return DEFER_OK;
}

int defer_stage_link(defer_stage_t prod, defer_stage_t cons) {
  DEFER_CHECK(prod && cons && prod != cons, "link: bad handles");
  DEFER_CHECK(!prod->finalized && !cons->finalized, "link: stage already finalized");
  if (prod->cfg.device != cons->cfg.device) {
    int can = 0;
    DEFER_CUDA(cudaDeviceCanAccessPeer(&can, prod->cfg.device, cons->cfg.device));
    DEFER_CHECK(can, "link: device %d cannot access device %d over P2P", prod->cfg.device, cons->cfg.device);
    DEFER_CUDA(cudaSetDevice(prod->cfg.device));
    cudaError_t e = cudaDeviceEnablePeerAccess(cons->cfg.device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) DEFER_CUDA(e);
    cudaGetLastError();
    DEFER_CUDA(cudaSetDevice(cons->cfg.device));
    e = cudaDeviceEnablePeerAccess(prod->cfg.device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) DEFER_CUDA(e);
    cudaGetLastError();
  }
  LinkToken tin, tout;
  fill_token(cons, 0, &tin);
  fill_token(prod, 1, &tout);
  DEFER_TRY(apply_token(prod, 0, &tin, cons->arena, false));
  DEFER_TRY(apply_token(cons, 1, &tout, prod->arena, false));
  return DEFER_OK;
}

int defer_stage_export_link(defer_stage_t s, int role, void* token) {
  DEFER_CHECK(s && token && (role == 0 || role == 1), "export_link: bad arguments");
  DEFER_TRY(set_device(s));
  LinkToken t;
  fill_token(s, role, &t);
  DEFER_CUDA(cudaIpcGetMemHandle(&t.ipc, s->arena));
  memset(token, 0, DEFER_LINK_TOKEN_BYTES);
  memcpy(token, &t, sizeof t);
  return DEFER_OK;
}

int defer_stage_import_link(defer_stage_t s, int role, const void* token) {
  DEFER_CHECK(s && token && (role == 0 || role == 1), "import_link: bad arguments");
  DEFER_CHECK(!s->finalized, "import_link: stage already finalized");
  LinkToken t;
  memcpy(&t, token, sizeof t);
  DEFER_CHECK(t.magic == TOKEN_MAGIC && t.role == role, "import_link: not a link token for role %d", role);
  DEFER_TRY(set_device(s));
  uint8_t* mapped = nullptr;
  bool is_ipc = false;
  if (t.pid == (int)getpid()) {
    mapped = (uint8_t*)(uintptr_t)t.local_base;  // same process: the pointer is already valid here
    if (t.device != s->cfg.device) {
      cudaError_t e = cudaDeviceEnablePeerAccess(t.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) DEFER_CUDA(e);
      cudaGetLastError();
    }
  } else {
    DEFER_CUDA(cudaIpcOpenMemHandle((void**)&mapped, t.ipc, cudaIpcMemLazyEnablePeerAccess));
    is_ipc = true;
  }
  return apply_token(s, role, &t, mapped, is_ipc);
}

int defer_stage_unlink(defer_stage_t s) {
  DEFER_CHECK(s, "unlink: null");
  DEFER_TRY(set_device(s));
  DEFER_CUDA(cudaDeviceSynchronize());
  if (s->cons_arena && s->cons_is_ipc) DEFER_CUDA(cudaIpcCloseMemHandle(s->cons_arena));
  if (s->prod_arena && s->prod_is_ipc) DEFER_CUDA(cudaIpcCloseMemHandle(s->prod_arena));
  s->cons_arena = nullptr;
  s->prod_arena = nullptr;
  s->cons_is_ipc = s->prod_is_ipc = false;
  s->unlinked = true;
  return DEFER_OK;
}

int defer_stage_finalize(defer_stage_t s) {
  DEFER_CHECK(s, "finalize: null");
  DEFER_CHECK(!s->finalized, "finalize: already done");
  DEFER_CHECK(s->cfg.is_first || s->has_prod, "finalize: stage is not first and has no producer link");
  DEFER_CHECK(s->cfg.is_last || s->has_cons, "finalize: stage is not last and has no consumer link");
  DEFER_TRY(set_device(s));
  // megakernel groups: maximal runs of consecutive wgmma convs (DEFER_MEGA=0 disables)
  s->op_group.assign(s->ops.size(), -1);
  {
    const char* e = getenv("DEFER_MEGA");
    const bool mega_on = e && atoi(e) != 0;   // cluster-chain megakernel: opt-in (wins only when launch-bound)
    int i = 0, n = (int)s->ops.size();
    while (mega_on && i < n) {
      // a conv carrying a folded AFFINE op ends a run and runs on its own (conv_mega_kernel has no second output)
      if (s->ops[i].backend != 2 || s->ops[i].aff_op >= 0) { ++i; continue; }
      int j = i;
      while (j + 1 < n && s->ops[j + 1].backend == 2 && s->ops[j + 1].aff_op < 0) ++j;
      if (j > i) {
        defer_stage_s::MegaGroup g;
        g.first = i;
        g.last = j;
        for (int k = i; k <= j; ++k) s->op_group[k] = (int)s->groups.size();
        s->groups.push_back(g);
      }
      i = j + 1;
    }
  }
  // wgmma conv plans need final buffer addresses (TMA tensor maps embed them)
  for (int oi = 0; oi < (int)s->ops.size(); ++oi) {
    OpRt& op = s->ops[oi];
    if (op.backend != 2 && op.backend != 4) continue;
    const defer_op_desc& d = op.d;
    const Buf& bi = s->bufs[d.in0];
    const Buf& bo = s->bufs[d.out];
    bool mega_plan = s->op_group[oi] >= 0;
    const bool stem = op.backend == 4;
    if (stem && !op.w_pad) {
      // [K, cout] filter bank (HWIO flattened) zero-padded to [k_pad, cout]
      const size_t kc = (size_t)d.kh * d.kw * bi.c * bo.c;
      DEFER_CUDA(cudaMalloc(&op.w_pad, (size_t)op.k_pad * bo.c * sizeof(float)));
      s->workspace.push_back(op.w_pad);
      DEFER_CUDA(cudaMemset(op.w_pad, 0, (size_t)op.k_pad * bo.c * sizeof(float)));
      DEFER_CUDA(cudaMemcpy(op.w_pad, s->d_weights[d.w_kernel], kc * sizeof(float), cudaMemcpyDeviceToDevice));
    }
    // Executor choice.  Ops of a megakernel group keep the group's 64-wide tiles.  Otherwise an op with enough output
    // tiles runs on the streaming persistent kernel (deep operand ring, overlapped in-place epilogue); small ops keep
    // the one-tile-per-CTA kernel (BN = 128 where C_out allows, split-K below 4 CTAs).
    //   DEFER_STREAM=0           -> the persistent grid with 64-wide N tiles only (launch_conv_persistent) instead
    //   DEFER_STREAM_MIN_TILES   -> threshold in 128 x 64 tiles (default 96)
    //   DEFER_STREAM_BN          -> force the N tile (64 | 128); default 128 whenever C_out % 128 == 0 (the A tile is
    //                               fetched once per N tile: wide N tiles halve the activation traffic;
    //                               DEFER_STREAM_BN128_TILES = minimum tile count to allow it)
    const int stream_on = getenv("DEFER_STREAM") ? atoi(getenv("DEFER_STREAM")) : 1;
    int stream_bn = 0;
    for (int attempt = 0; attempt < 2; ++attempt) {
      if (stem)   // 1x1 conv over the patch matrix: "image" = output grid, channels = k_pad
        DEFER_TRY(umma_conv_prepare(&op.umma, s->cfg.fmt, s->cfg.batch, bo.h, bo.w, op.k_pad, bo.h, bo.w, bo.c, 1, 1, 1, 1, 0, 0,
                                    d.flags, (const float*)op.w_pad,
                                    d.w_scale >= 0 ? (const float*)s->d_weights[d.w_scale] : nullptr,
                                    d.w_shift >= 0 ? (const float*)s->d_weights[d.w_shift] : nullptr, mega_plan, stream_bn));
      else
      DEFER_TRY(umma_conv_prepare(&op.umma, s->cfg.fmt, s->cfg.batch, bi.h, bi.w, bi.c, bo.h, bo.w, bo.c, d.kh, d.kw, d.sh,
                                  d.sw, d.pad_t, d.pad_l, d.flags, (const float*)s->d_weights[d.w_kernel],
                                  d.w_scale >= 0 ? (const float*)s->d_weights[d.w_scale] : nullptr,
                                  d.w_shift >= 0 ? (const float*)s->d_weights[d.w_shift] : nullptr, mega_plan, stream_bn));
      const int m_tiles = op.umma.m_tiles;
      op.n_tiles64 = m_tiles * (bo.c / 64);
      op.persist = (mega_plan || stream_bn > 0) && s->op_group[oi] < 0;
      if (attempt == 0 && !mega_plan) {
        const char* pe = getenv(stream_on ? "DEFER_STREAM_MIN_TILES" : "DEFER_PERSIST_MIN_TILES");
        const int min_tiles = pe ? atoi(pe) : (stream_on ? 96 : 192);
        if (min_tiles > 0 && op.n_tiles64 >= min_tiles) {
          umma_conv_release(op.umma);   // many tiles: re-plan for a persistent grid (whole K loop per tile, no split-K)
          if (stream_on) {
            const char* fb = getenv("DEFER_STREAM_BN");
            const char* mt = getenv("DEFER_STREAM_BN128_TILES");
            const int min128 = mt ? atoi(mt) : 1;
            stream_bn = (bo.c % 128 == 0 && m_tiles * (bo.c / 128) >= min128) ? 128 : 64;
            if (fb && (atoi(fb) == 64 || (atoi(fb) == 128 && bo.c % 128 == 0))) stream_bn = atoi(fb);
          } else {
            mega_plan = true;
          }
          continue;
        }
      }
      break;
    }
    op.stream = op.persist && stream_bn > 0;
    if (op.persist && op.aff_op >= 0) op.kname = op.stream ? "conv_stream_aff_kernel" : "conv_stream_aff_kernel(grid)";
    else if (op.persist) op.kname = std::string(stem ? "stem_im2col+" : "") + (op.stream ? "conv_stream_kernel" : "conv_mega_kernel(grid)");
    if (op.aff_op >= 0) {
      const defer_op_desc& a = s->ops[op.aff_op].d;
      op.umma.aff = true;
      op.umma.scale2 = (const float*)s->d_weights[a.w_scale];
      op.umma.shift2 = (const float*)s->d_weights[a.w_shift];
      op.umma.relu2 = (a.flags & DEFER_FLAG_RELU) ? 1 : 0;
      op.umma.store_first = op.store_out ? 1 : 0;
      s->ops[op.aff_op].kname = "affine (fused into " + op.kname + ")";
    }
    // fused stem: no patch matrix at all when the tile geometry allows it and the output stays on this GPU
    {
      const int fuse = getenv("DEFER_STEM_FUSED") ? atoi(getenv("DEFER_STEM_FUSED")) : 1;
      const bool out_local = s->hop == HOP_COPY || !((d.out == s->cfg.output_buf) && !s->cfg.is_last);
      op.stem_fused = stem && fuse && op.stream && op.umma.bn == 64 && out_local &&
                      umma_stem_fusable(s->cfg.fmt, bi.c, bo.h, bo.w, bo.c, d.kh, d.kw, d.sh, d.sw, d.flags);
      if (op.stem_fused) {
        op.kname = "conv_stem_kernel";
        op.n_kernels = 1;
      }
    }
    for (int l = 0; l < s->cfg.depth; ++l) {
      Lane& L = s->lanes[l];
      // the stage output of a non-last stage is the next GPU's input slot: plain stores over NVLink
      L.umma[oi].direct_out = (d.out == s->cfg.output_buf) && !s->cfg.is_last && s->hop == HOP_DIRECT;
      const void* conv_in = L.buf[d.in0];
      if (stem) {
        if (L.im2col.size() < s->ops.size()) L.im2col.resize(s->ops.size(), nullptr);
        if (!L.im2col[oi] && !op.stem_fused) {
          const size_t bytes = (size_t)s->cfg.batch * bo.h * bo.w * op.k_pad * fmt_bytes_per_elem(s->cfg.fmt);
          DEFER_CUDA(cudaMalloc(&L.im2col[oi], bytes));
          s->workspace.push_back(L.im2col[oi]);
        }
        conv_in = op.stem_fused ? L.buf[d.out] : L.im2col[oi];   // fused: the A tensor map is never used (any valid pointer)
      }
      DEFER_TRY(umma_conv_bind(op.umma, &L.umma[oi], conv_in,
                               (d.flags & DEFER_FLAG_RESIDUAL) ? L.buf[d.in1] : nullptr, L.buf[d.out]));
      if (op.aff_op >= 0) L.umma[oi].y2 = L.buf[s->ops[op.aff_op].d.out];
    }
  }
  // Fold a PREPROCESS op into the fused stem conv when that conv is the only reader of its (non-output) F32 image:
  // the stem then reads the uint8 image and preprocesses each value of its image window itself.  Every other path runs
  // preprocess_kernel (preprocess_tf_kernel in tf mode).
  for (int pi = 0; pi < (int)s->ops.size(); ++pi) {
    OpRt& pre = s->ops[pi];
    if (pre.d.kind != DEFER_OP_PREPROCESS || pre.d.out == s->cfg.output_buf) continue;
    int reader = -1, n_reads = 0;
    for (int oi = 0; oi < (int)s->ops.size(); ++oi) {
      const defer_op_desc& d = s->ops[oi].d;
      const int r = (d.in0 == pre.d.out) + (d.in1 == pre.d.out);
      if (r) reader = oi;
      n_reads += r;
    }
    if (n_reads != 1 || s->ops[reader].d.kind != DEFER_OP_CONV || !s->ops[reader].stem_fused) continue;
    OpRt& conv = s->ops[reader];
    pre.folded_into = reader;
    pre.n_kernels = 0;
    pre.alg_bytes = 0;
    conv.u8_pre = pi;
    conv.kname = pre.d.mode == DEFER_PRE_TF ? "conv_stem_u8tf_kernel" : "conv_stem_u8_kernel";
    pre.kname = "preprocess (fused into " + conv.kname + ")";
    conv.alg_bytes -= (double)s->bufs[pre.d.in0].elems * 3.0;   // the image is read at 1 B/elem instead of 4
  }
  for (int oi = 0; oi < (int)s->ops.size(); ++oi) {
    OpRt& op = s->ops[oi];
    if ((op.backend != 2 && op.backend != 4) || !op.persist) continue;
    const size_t ob = umma_mega_op_bytes();
    std::vector<uint8_t> host(ob);
    for (int l = 0; l < s->cfg.depth; ++l) {
      Lane& L = s->lanes[l];
      L.persist_op.resize(s->ops.size(), nullptr);
      DEFER_TRY(umma_mega_fill(host.data(), op.umma, L.umma[oi]));
      if (op.stem_fused) {
        const defer_op_desc& d = op.d;
        const Buf& bi = s->bufs[d.in0];
        op.stem_tiles = umma_mega_set_stem(host.data(), (const float*)L.buf[d.in0], bi.h, bi.w, bi.c, d.kh, d.kw, d.sh, d.sw,
                                           d.pad_t, d.pad_l);
        if (op.u8_pre >= 0) {
          const OpRt& pre = s->ops[op.u8_pre];
          umma_mega_set_stem_u8(host.data(), (const uint8_t*)L.buf[pre.d.in0], pre.pre_shift);
        }
      }
      DEFER_CUDA(cudaMalloc(&L.persist_op[oi], ob));
      s->workspace.push_back(L.persist_op[oi]);
      DEFER_CUDA(cudaMemcpy(L.persist_op[oi], host.data(), ob, cudaMemcpyHostToDevice));
    }
  }
  for (auto& g : s->groups) {
    const int n = g.last - g.first + 1;
    const size_t ob = umma_mega_op_bytes();
    std::vector<uint8_t> host(ob * n);
    g.dev_ops.assign(s->cfg.depth, nullptr);
    for (int l = 0; l < s->cfg.depth; ++l) {
      for (int k = 0; k < n; ++k)
        DEFER_TRY(umma_mega_fill(host.data() + ob * k, s->ops[g.first + k].umma, s->lanes[l].umma[g.first + k]));
      DEFER_CUDA(cudaMalloc(&g.dev_ops[l], ob * n));
      s->workspace.push_back(g.dev_ops[l]);
      DEFER_CUDA(cudaMemcpy(g.dev_ops[l], host.data(), ob * n, cudaMemcpyHostToDevice));
    }
  }
  DEFER_CUDA(cudaDeviceSynchronize());
  if (s->cfg.use_graph) {
    for (int l = 0; l < s->cfg.depth; ++l) {
      Lane& L = s->lanes[l];
      DEFER_CUDA(cudaStreamBeginCapture(L.stream, cudaStreamCaptureModeThreadLocal));
      int rc = enqueue_lane(s, l, L.stream);
      cudaError_t e = cudaStreamEndCapture(L.stream, &L.graph);
      if (rc != DEFER_OK) return rc;
      DEFER_CUDA(e);
      DEFER_CUDA(cudaGraphInstantiate(&L.exec, L.graph, 0));
    }
  }
  s->finalized = true;
  return DEFER_OK;
}

// ------------------------------------------------------------------------------------------ steady state
int defer_stage_submit(defer_stage_t s, uint64_t seq, const void* host_in, uint64_t nbytes) {
  DEFER_CHECK(s && host_in, "submit: null");
  DEFER_CHECK(s->cfg.is_first, "submit: only the first stage takes host input");
  DEFER_CHECK(s->dec.op < 0, "submit: this stage takes %s files (defer_stage_submit_%ss)", dec_name(s, true),
              dec_name(s, false));
  DEFER_CHECK(s->frames.op_w < 0, "submit: this stage takes images of mixed sizes (defer_stage_submit_frames)");
  const Buf& b = s->bufs[s->cfg.input_buf];
  DEFER_CHECK(nbytes == b.bytes, "submit: got %llu bytes, stage input is %zu", (unsigned long long)nbytes, b.bytes);
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  DEFER_CUDA(cudaMemcpyAsync(L.buf[s->cfg.input_buf], host_in, nbytes, cudaMemcpyHostToDevice, L.stream));
  return DEFER_OK;
}

int defer_stage_submit_part(defer_stage_t s, uint64_t seq, int index, int count, const void* host_in, uint64_t nbytes) {
  DEFER_CHECK(s && host_in, "submit_part: null");
  DEFER_CHECK(s->cfg.is_first, "submit_part: only the first stage takes host input");
  DEFER_CHECK(s->dec.op < 0, "submit_part: this stage takes %s files (defer_stage_submit_%ss)", dec_name(s, true),
              dec_name(s, false));
  DEFER_CHECK(s->frames.op_w < 0, "submit_part: this stage takes images of mixed sizes (defer_stage_submit_frames)");
  const Buf& b = s->bufs[s->cfg.input_buf];
  const size_t sample = b.bytes / (size_t)s->cfg.batch;       // first-stage input is plain fp32 NHWC: samples are contiguous
  DEFER_CHECK(index >= 0 && count >= 1 && index + count <= s->cfg.batch, "submit_part: samples [%d, %d) outside the microbatch of %d",
              index, index + count, s->cfg.batch);
  DEFER_CHECK(nbytes == sample * (size_t)count, "submit_part: got %llu bytes, %d sample(s) are %zu", (unsigned long long)nbytes,
              count, sample * (size_t)count);
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  DEFER_CUDA(cudaMemcpyAsync((uint8_t*)L.buf[s->cfg.input_buf] + sample * (size_t)index, host_in, nbytes, cudaMemcpyHostToDevice,
                             L.stream));
  return DEFER_OK;
}

int defer_stage_submit_parts(defer_stage_t s, uint64_t seq, int first_index, int n_items, int samples_per_item,
                             const void* const* host_ptrs, uint64_t nbytes_per_item) {
  DEFER_CHECK(s && host_ptrs && n_items >= 1 && samples_per_item >= 1, "submit_parts: bad arguments");
  DEFER_CHECK(s->cfg.is_first, "submit_parts: only the first stage takes host input");
  DEFER_CHECK(s->dec.op < 0, "submit_parts: this stage takes %s files (defer_stage_submit_%ss)", dec_name(s, true),
              dec_name(s, false));
  DEFER_CHECK(s->frames.op_w < 0, "submit_parts: this stage takes images of mixed sizes (defer_stage_submit_frames)");
  const Buf& b = s->bufs[s->cfg.input_buf];
  const size_t sample = b.bytes / (size_t)s->cfg.batch;
  DEFER_CHECK(first_index >= 0 && first_index + n_items * samples_per_item <= s->cfg.batch,
              "submit_parts: samples [%d, %d) outside the microbatch of %d", first_index, first_index + n_items * samples_per_item,
              s->cfg.batch);
  DEFER_CHECK(nbytes_per_item == sample * (size_t)samples_per_item, "submit_parts: items are %llu bytes, %d sample(s) are %zu",
              (unsigned long long)nbytes_per_item, samples_per_item, sample * (size_t)samples_per_item);
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  uint8_t* dst = (uint8_t*)L.buf[s->cfg.input_buf] + sample * (size_t)first_index;
  for (int i = 0; i < n_items; ++i) {
    DEFER_CHECK(host_ptrs[i], "submit_parts: item %d is null", i);
    DEFER_CUDA(cudaMemcpyAsync(dst + (size_t)i * nbytes_per_item, host_ptrs[i], nbytes_per_item, cudaMemcpyHostToDevice, L.stream));
  }
  return DEFER_OK;
}

int defer_stage_submit_frames(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* images,
                              const int32_t* hw, const int32_t* tables, uint64_t table_bytes) {
  DEFER_CHECK(s && images && hw && tables && n >= 1, "submit_frames: bad arguments");
  DEFER_CHECK(s->cfg.is_first, "submit_frames: only the first stage takes host input");
  const auto& f = s->frames;
  DEFER_CHECK(f.op_w >= 0, "submit_frames: the stage takes one image size (no DEFER_RESIZE_SAMPLE_* ops); use defer_stage_submit*");
  DEFER_CHECK(s->dec.op < 0, "submit_frames: this stage takes %s files (defer_stage_submit_%ss)", dec_name(s, true),
              dec_name(s, false));
  DEFER_CHECK(first_index >= 0 && first_index <= s->cfg.batch - n, "submit_frames: samples [%d, %d) outside the microbatch of %d",
              first_index, first_index + n, s->cfg.batch);
  DEFER_CHECK(table_bytes == (uint64_t)n * f.block_ints * 4, "submit_frames: got %llu table bytes, %d blocks are %zu",
              (unsigned long long)table_bytes, n, (size_t)n * f.block_ints * 4);
  for (int i = 0; i < n; ++i) {   // all checks first: a refused call copies nothing
    const int h = hw[2 * i], w = hw[2 * i + 1];
    const int32_t* blk = tables + (size_t)i * f.block_ints;
    DEFER_CHECK(images[i], "submit_frames: image %d is null", i);
    DEFER_CHECK(h >= 1 && h <= f.H && w >= 1 && w <= f.W, "submit_frames: image %d is %dx%d, the slot takes 1..%d x 1..%d", i, h,
                w, f.H, f.W);
    DEFER_CHECK(blk[0] == h && blk[1] == w, "submit_frames: table block %d is for %dx%d, image %d is %dx%d", i, blk[0], blk[1], i,
                h, w);
  }
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  const size_t sample = (size_t)f.H * f.W * 3;
  uint8_t* slot = (uint8_t*)L.buf[s->cfg.input_buf];
  for (int i = 0; i < n; ++i)   // the image's own bytes only, packed at the start of its sample slot
    DEFER_CUDA(cudaMemcpyAsync(slot + (size_t)(first_index + i) * sample, images[i], (size_t)hw[2 * i] * hw[2 * i + 1] * 3,
                               cudaMemcpyHostToDevice, L.stream));
  DEFER_CUDA(cudaMemcpyAsync(L.tables + (size_t)first_index * f.block_ints, tables, table_bytes, cudaMemcpyHostToDevice, L.stream));
  return DEFER_OK;
}

}  // extern "C"

namespace defer {

// The checks of one JPEG file of a submit call (`who` names it in the messages): its size within 4..slot, its block's
// size within the bound and equal to its resize block's, and its entropy data inside the file.
static int check_jpeg_file(const char* who, const defer_stage_s* s, int i, uint64_t nbytes, uint64_t slot, const int32_t* rb,
                           const int32_t* jb) {
  const auto& f = s->frames;
  DEFER_CHECK(nbytes >= 4 && nbytes <= slot, "%s: file %d has %llu bytes, the slot takes 4..%llu", who, i,
              (unsigned long long)nbytes, (unsigned long long)slot);
  DEFER_CHECK(jb[0] >= 1 && jb[0] <= f.H && jb[1] >= 1 && jb[1] <= f.W, "%s: file %d is %dx%d, the slot takes 1..%d x "
              "1..%d", who, i, jb[0], jb[1], f.H, f.W);
  DEFER_CHECK(rb[0] == jb[0] && rb[1] == jb[1], "%s: resize block %d is for %dx%d, JPEG block %d for %dx%d", who, i, rb[0],
              rb[1], i, jb[0], jb[1]);
  DEFER_CHECK(jb[6] >= 0 && jb[7] >= 0 && (uint64_t)jb[6] + (uint64_t)jb[7] <= nbytes,
              "%s: file %d: entropy data [%d, %d + %d) outside its %llu bytes", who, i, jb[6], jb[6], jb[7],
              (unsigned long long)nbytes);
  DEFER_CHECK(jb[10] >= 0 && jb[10] <= DEFER_JPEG_MAX_SCANS && jb[11] >= 0 && jb[11] <= DEFER_JPEG_MAX_TABLES,
              "%s: file %d: %d scans and %d Huffman tables, at most %d and %d", who, i, jb[10], jb[11],
              DEFER_JPEG_MAX_SCANS, DEFER_JPEG_MAX_TABLES);
  for (int k = 0; k < jb[10]; ++k) {
    const int32_t* sc = jb + DEFER_JPEG_SCAN_OFF + k * DEFER_JPEG_SCAN_INTS;
    DEFER_CHECK(sc[9] >= 0 && sc[10] >= 0 && (uint64_t)sc[9] + (uint64_t)sc[10] <= nbytes,
                "%s: file %d: scan %d's entropy data [%d, %d + %d) outside its %llu bytes", who, i, k, sc[9], sc[9],
                sc[10], (unsigned long long)nbytes);
  }
  return DEFER_OK;
}

// the prefix of a checked JPEG block that its file uses: a baseline file's DEFER_JPEG_BASE_INTS, a progressive one's pool
static size_t jpeg_used_ints(const int32_t* jb) {
  return jb[10] ? (size_t)DEFER_JPEG_POOL_OFF + (size_t)jb[11] * DEFER_JPEG_HUFF_INTS : (size_t)DEFER_JPEG_BASE_INTS;
}

// The checks of one PNG file of a submit call: its size within 8..slot, its block's size within the bound and equal to
// its resize block's, its row length and filter unit those of its size, colour type and depth, and its IDAT chunks
// inside the file and summing to its stream length.
static int check_png_file(const char* who, const defer_stage_s* s, int i, uint64_t nbytes, uint64_t slot, const int32_t* rb,
                          const int32_t* pb) {
  const auto& f = s->frames;
  DEFER_CHECK(nbytes >= 8 && nbytes <= slot, "%s: file %d has %llu bytes, the slot takes 8..%llu", who, i,
              (unsigned long long)nbytes, (unsigned long long)slot);
  DEFER_CHECK(pb[0] >= 1 && pb[0] <= f.H && pb[1] >= 1 && pb[1] <= f.W, "%s: file %d is %dx%d, the slot takes 1..%d x "
              "1..%d", who, i, pb[0], pb[1], f.H, f.W);
  DEFER_CHECK(rb[0] == pb[0] && rb[1] == pb[1], "%s: resize block %d is for %dx%d, PNG block %d for %dx%d", who, i, rb[0],
              rb[1], i, pb[0], pb[1]);
  const int ct = pb[2], d = pb[3];
  const int ch = ct == 0 ? 1 : ct == 2 ? 3 : ct == 3 ? 1 : ct == 4 ? 2 : ct == 6 ? 4 : 0;
  const bool depth_ok = d == 8 || (d == 16 && ct != 3) || ((d == 1 || d == 2 || d == 4) && (ct == 0 || ct == 3));
  DEFER_CHECK(ch && depth_ok && pb[4] == (int)(((int64_t)pb[1] * ch * d + 7) / 8) && pb[5] == std::max(1, ch * d / 8),
              "%s: file %d: colour type %d, depth %d, %d bytes per row and filter unit %d do not match", who, i, ct, d,
              pb[4], pb[5]);
  DEFER_CHECK(pb[6] >= 1 && pb[6] <= DEFER_PNG_MAX_IDAT && pb[8] >= 0 && pb[8] <= 256,
              "%s: file %d: %d IDAT chunks (1..%d) and %d palette entries (0..256)", who, i, pb[6], DEFER_PNG_MAX_IDAT,
              pb[8]);
  int64_t total = 0;
  for (int k = 0; k < pb[6]; ++k) {
    const int32_t off = pb[DEFER_PNG_IDAT_OFF + 2 * k], len = pb[DEFER_PNG_IDAT_OFF + 2 * k + 1];
    DEFER_CHECK(off >= 0 && len >= 0 && (uint64_t)off + (uint64_t)len <= nbytes,
                "%s: file %d: IDAT chunk %d [%d, %d + %d) outside its %llu bytes", who, i, k, off, off, len,
                (unsigned long long)nbytes);
    total += len;
  }
  DEFER_CHECK(total == pb[7], "%s: file %d: its IDAT chunks hold %lld bytes, its block says %d", who, i, (long long)total,
              pb[7]);
  return DEFER_OK;
}

// the prefix of a checked PNG block that its file uses: header, palette and its IDAT ranges
static size_t png_used_ints(const int32_t* pb) { return (size_t)DEFER_PNG_IDAT_OFF + 2 * (size_t)pb[6]; }

}  // namespace defer

extern "C" {

int defer_stage_submit_jpegs(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                             const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes) {
  DEFER_CHECK(s && data && nbytes && blocks && n >= 1, "submit_jpegs: bad arguments");
  DEFER_CHECK(s->cfg.is_first, "submit_jpegs: only the first stage takes host input");
  DEFER_CHECK(s->dec.kind == DEFER_OP_JPEG_DECODE, "submit_jpegs: the stage has no DEFER_OP_JPEG_DECODE op");
  const auto& f = s->frames;
  DEFER_CHECK(first_index >= 0 && first_index <= s->cfg.batch - n, "submit_jpegs: samples [%d, %d) outside the microbatch of %d",
              first_index, first_index + n, s->cfg.batch);
  const size_t per = f.block_ints + DEFER_JPEG_BLOCK_INTS;     // one file's resize block, then its JPEG block
  DEFER_CHECK(block_bytes == (uint64_t)n * per * 4, "submit_jpegs: got %llu block bytes, %d files take %zu",
              (unsigned long long)block_bytes, n, (size_t)n * per * 4);
  const uint64_t slot = (uint64_t)f.H * f.W * 3;
  for (int i = 0; i < n; ++i) {   // all checks first: a refused call copies nothing
    const int32_t* rb = blocks + (size_t)i * per;
    DEFER_CHECK(data[i], "submit_jpegs: file %d is null", i);
    DEFER_TRY(check_jpeg_file("submit_jpegs", s, i, nbytes[i], slot, rb, rb + f.block_ints));
  }
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  uint8_t* dst = (uint8_t*)L.buf[s->cfg.input_buf];
  for (int i = 0; i < n; ++i)   // the file's own bytes only, at the start of its sample slot
    DEFER_CUDA(cudaMemcpyAsync(dst + (size_t)(first_index + i) * slot, data[i], nbytes[i], cudaMemcpyHostToDevice, L.stream));
  DEFER_CUDA(cudaMemcpy2DAsync(L.tables + (size_t)first_index * f.block_ints, f.block_ints * 4, blocks, per * 4,
                               f.block_ints * 4, n, cudaMemcpyHostToDevice, L.stream));
  // each JPEG block's prefix that its file uses (a baseline file: DEFER_JPEG_BASE_INTS), in one copy when all are baseline
  auto used = [&](int i) { return jpeg_used_ints(blocks + (size_t)i * per + f.block_ints); };
  bool all_base = true;
  for (int i = 0; i < n; ++i) all_base &= used(i) == DEFER_JPEG_BASE_INTS;
  if (all_base) {
    DEFER_CUDA(cudaMemcpy2DAsync(L.dec_blocks + (size_t)first_index * DEFER_JPEG_BLOCK_INTS, DEFER_JPEG_BLOCK_INTS * 4,
                                 blocks + f.block_ints, per * 4, DEFER_JPEG_BASE_INTS * 4, n, cudaMemcpyHostToDevice,
                                 L.stream));
  } else {
    for (int i = 0; i < n; ++i)
      DEFER_CUDA(cudaMemcpyAsync(L.dec_blocks + (size_t)(first_index + i) * DEFER_JPEG_BLOCK_INTS,
                                 blocks + (size_t)i * per + f.block_ints, used(i) * 4, cudaMemcpyHostToDevice, L.stream));
  }
  return DEFER_OK;
}

int defer_stage_submit_pngs(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                            const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes) {
  DEFER_CHECK(s && data && nbytes && blocks && n >= 1, "submit_pngs: bad arguments");
  DEFER_CHECK(s->cfg.is_first, "submit_pngs: only the first stage takes host input");
  DEFER_CHECK(s->dec.kind == DEFER_OP_PNG_DECODE, "submit_pngs: the stage has no DEFER_OP_PNG_DECODE op");
  const auto& f = s->frames;
  DEFER_CHECK(first_index >= 0 && first_index <= s->cfg.batch - n, "submit_pngs: samples [%d, %d) outside the microbatch of %d",
              first_index, first_index + n, s->cfg.batch);
  const size_t per = f.block_ints + DEFER_PNG_BLOCK_INTS;      // one file's resize block, then its PNG block
  DEFER_CHECK(block_bytes == (uint64_t)n * per * 4, "submit_pngs: got %llu block bytes, %d files take %zu",
              (unsigned long long)block_bytes, n, (size_t)n * per * 4);
  const uint64_t slot = DEFER_PNG_SLOT_BYTES((uint64_t)f.H, (uint64_t)f.W);
  for (int i = 0; i < n; ++i) {   // all checks first: a refused call copies nothing
    const int32_t* rb = blocks + (size_t)i * per;
    DEFER_CHECK(data[i], "submit_pngs: file %d is null", i);
    DEFER_TRY(check_png_file("submit_pngs", s, i, nbytes[i], slot, rb, rb + f.block_ints));
  }
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  uint8_t* dst = (uint8_t*)L.buf[s->cfg.input_buf];
  for (int i = 0; i < n; ++i)   // the file's own bytes only, at the start of its sample slot
    DEFER_CUDA(cudaMemcpyAsync(dst + (size_t)(first_index + i) * slot, data[i], nbytes[i], cudaMemcpyHostToDevice, L.stream));
  DEFER_CUDA(cudaMemcpy2DAsync(L.tables + (size_t)first_index * f.block_ints, f.block_ints * 4, blocks, per * 4,
                               f.block_ints * 4, n, cudaMemcpyHostToDevice, L.stream));
  for (int i = 0; i < n; ++i) {   // each PNG block's prefix that its file uses: header, palette and its IDAT ranges
    const int32_t* pb = blocks + (size_t)i * per + f.block_ints;
    DEFER_CUDA(cudaMemcpyAsync(L.dec_blocks + (size_t)(first_index + i) * DEFER_PNG_BLOCK_INTS, pb, png_used_ints(pb) * 4,
                               cudaMemcpyHostToDevice, L.stream));
  }
  return DEFER_OK;
}

int defer_stage_submit_images(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                              const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes) {
  DEFER_CHECK(s && data && nbytes && blocks && n >= 1, "submit_images: bad arguments");
  DEFER_CHECK(s->cfg.is_first, "submit_images: only the first stage takes host input");
  DEFER_CHECK(s->dec.kind == DEFER_OP_IMAGE_DECODE, "submit_images: the stage has no DEFER_OP_IMAGE_DECODE op");
  const auto& f = s->frames;
  DEFER_CHECK(first_index >= 0 && first_index <= s->cfg.batch - n, "submit_images: samples [%d, %d) outside the microbatch of %d",
              first_index, first_index + n, s->cfg.batch);
  const size_t per = f.block_ints + DEFER_IMAGE_BLOCK_INTS;    // one file's resize block, then its tagged block
  DEFER_CHECK(block_bytes == (uint64_t)n * per * 4, "submit_images: got %llu block bytes, %d files take %zu",
              (unsigned long long)block_bytes, n, (size_t)n * per * 4);
  const uint64_t slot = DEFER_PNG_SLOT_BYTES((uint64_t)f.H, (uint64_t)f.W);
  const uint64_t jpeg_slot = (uint64_t)f.H * f.W * 3;          // a JPEG's bit positions are ints (jpeg_bound_ok)
  for (int i = 0; i < n; ++i) {   // all checks first: a refused call copies nothing
    const int32_t* rb = blocks + (size_t)i * per;
    const int32_t* b = rb + f.block_ints;
    DEFER_CHECK(data[i], "submit_images: file %d is null", i);
    DEFER_CHECK(b[DEFER_IMAGE_TAG] == DEFER_IMAGE_JPEG || b[DEFER_IMAGE_TAG] == DEFER_IMAGE_PNG,
                "submit_images: file %d: block tag %d, neither DEFER_IMAGE_JPEG (%d) nor DEFER_IMAGE_PNG (%d)", i,
                b[DEFER_IMAGE_TAG], DEFER_IMAGE_JPEG, DEFER_IMAGE_PNG);
    if (b[DEFER_IMAGE_TAG] == DEFER_IMAGE_JPEG)
      DEFER_TRY(check_jpeg_file("submit_images", s, i, nbytes[i], jpeg_slot, rb, b));
    else
      DEFER_TRY(check_png_file("submit_images", s, i, nbytes[i], slot, rb, b));
  }
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[seq % s->cfg.depth];
  uint8_t* dst = (uint8_t*)L.buf[s->cfg.input_buf];
  for (int i = 0; i < n; ++i)   // the file's own bytes only, at the start of its sample slot
    DEFER_CUDA(cudaMemcpyAsync(dst + (size_t)(first_index + i) * slot, data[i], nbytes[i], cudaMemcpyHostToDevice, L.stream));
  DEFER_CUDA(cudaMemcpy2DAsync(L.tables + (size_t)first_index * f.block_ints, f.block_ints * 4, blocks, per * 4,
                               f.block_ints * 4, n, cudaMemcpyHostToDevice, L.stream));
  for (int i = 0; i < n; ++i) {   // each block's prefix that its file uses, in its format's layout (the tag is in both)
    const int32_t* b = blocks + (size_t)i * per + f.block_ints;
    const size_t used = b[DEFER_IMAGE_TAG] == DEFER_IMAGE_JPEG ? jpeg_used_ints(b) : png_used_ints(b);
    DEFER_CUDA(cudaMemcpyAsync(L.dec_blocks + (size_t)(first_index + i) * DEFER_IMAGE_BLOCK_INTS, b, used * 4,
                               cudaMemcpyHostToDevice, L.stream));
  }
  return DEFER_OK;
}

int defer_stage_step(defer_stage_t s, uint64_t seq) {
  DEFER_CHECK(s, "step: null");
  DEFER_CHECK(s->finalized, "step: call defer_stage_finalize first");
  DEFER_CHECK(!s->unlinked, "step: stage was unlinked");
  DEFER_TRY(set_device(s));
  int lane = (int)(seq % s->cfg.depth);
  Lane& L = s->lanes[lane];
  if (L.timed) DEFER_CUDA(cudaEventRecord(L.t0, L.stream));
  if (L.exec) {
    DEFER_CUDA(cudaGraphLaunch(L.exec, L.stream));
  } else {
    DEFER_TRY(enqueue_lane(s, lane, L.stream));
  }
  if (L.timed) DEFER_CUDA(cudaEventRecord(L.t1, L.stream));
  if (s->cfg.is_last) DEFER_CUDA(cudaEventRecord(L.done, L.stream));
  L.stepped = true;
  L.last_seq = seq;
  return DEFER_OK;
}

int defer_stage_status(defer_stage_t s) {
  DEFER_CHECK(s, "status: null");
  DEFER_TRY(set_device(s));
  int st = 0;
  DEFER_CUDA(cudaMemcpy(&st, s->status_ptr(), sizeof(int), cudaMemcpyDeviceToHost));
  if (st != 0) {
    set_error("device-side flag wait timed out on device %d (peer stage stalled or dead)", s->cfg.device);
    return DEFER_ERR_TIMEOUT;
  }
  return DEFER_OK;
}

int defer_stage_result(defer_stage_t s, uint64_t seq, void* host_out, uint64_t nbytes) {
  DEFER_CHECK(s && host_out, "result: null");
  DEFER_CHECK(s->cfg.is_last, "result: only the last stage returns results");
  const Buf& b = s->bufs[s->cfg.output_buf];
  DEFER_CHECK(nbytes == b.elems * 4, "result: got %llu bytes, stage output is %zu", (unsigned long long)nbytes, b.elems * 4);
  const int lane = (int)(seq % s->cfg.depth);
  Lane& L = s->lanes[lane];
  // the lane's one output buffer holds only its latest microbatch: a later step on it has overwritten seq's output
  if (!L.stepped || L.last_seq < seq) {
    set_error("result: microbatch %llu was never stepped (lane %d last ran %s%llu)", (unsigned long long)seq, lane,
              L.stepped ? "microbatch " : "nothing, ", (unsigned long long)L.last_seq);
    return DEFER_ERR_STATE;
  }
  if (L.last_seq != seq) {
    set_error("result: microbatch %llu is gone: lane %d has since run microbatch %llu over it (at most depth = %d microbatches "
              "may be between step and result)", (unsigned long long)seq, lane, (unsigned long long)L.last_seq, s->cfg.depth);
    return DEFER_ERR_STATE;
  }
  DEFER_TRY(set_device(s));
  DEFER_CUDA(cudaEventSynchronize(L.done));
  if (*reinterpret_cast<volatile int*>(L.status_host) != 0) {
    set_error("device-side flag wait timed out on device %d (upstream stage stalled or dead)", s->cfg.device);
    return DEFER_ERR_TIMEOUT;
  }
  memcpy(host_out, L.out_host, nbytes);
  return DEFER_OK;
}

int defer_stage_predict(defer_stage_t s, const void* host_in, uint64_t in_bytes, void* host_out, uint64_t out_bytes) {
  DEFER_CHECK(s && s->cfg.is_first && s->cfg.is_last, "predict: needs a single-stage pipeline");
  DEFER_TRY(defer_stage_submit(s, 0, host_in, in_bytes));
  DEFER_TRY(defer_stage_step(s, 0));
  return defer_stage_result(s, 0, host_out, out_bytes);
}

int defer_stage_sync(defer_stage_t s) {
  DEFER_CHECK(s, "sync: null");
  DEFER_TRY(set_device(s));
  for (auto& L : s->lanes) DEFER_CUDA(cudaStreamSynchronize(L.stream));
  return DEFER_OK;
}

int defer_stage_last_step_us(defer_stage_t s, int lane, float* us) {
  DEFER_CHECK(s && us && lane >= 0 && lane < s->cfg.depth, "last_step_us: bad arguments");
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[lane];
  if (!L.timed) {  // first call arms timing for subsequent steps
    L.timed = true;
    *us = -1.f;
    return DEFER_OK;
  }
  DEFER_CUDA(cudaEventSynchronize(L.t1));
  float ms = 0.f;
  DEFER_CUDA(cudaEventElapsedTime(&ms, L.t0, L.t1));
  *us = ms * 1000.f;
  return DEFER_OK;
}

int defer_stage_timer_start(defer_stage_t s) {
  DEFER_CHECK(s, "timer_start: null");
  DEFER_TRY(set_device(s));
  if (!s->job_t0) {
    DEFER_CUDA(cudaEventCreate(&s->job_t0));
    DEFER_CUDA(cudaEventCreate(&s->job_t1));
  }
  DEFER_CUDA(cudaEventRecord(s->job_t0, s->lanes[0].stream));
  return DEFER_OK;
}

int defer_stage_timer_stop(defer_stage_t s, float* ms) {
  DEFER_CHECK(s && ms, "timer_stop: null");
  DEFER_CHECK(s->job_t0, "timer_stop: timer_start was not called");
  DEFER_TRY(set_device(s));
  cudaStream_t s0 = s->lanes[0].stream;
  for (size_t l = 1; l < s->lanes.size(); ++l) {
    DEFER_CUDA(cudaEventRecord(s->lanes[l].join, s->lanes[l].stream));
    DEFER_CUDA(cudaStreamWaitEvent(s0, s->lanes[l].join, 0));
  }
  DEFER_CUDA(cudaEventRecord(s->job_t1, s0));
  DEFER_CUDA(cudaEventSynchronize(s->job_t1));
  DEFER_CUDA(cudaEventElapsedTime(ms, s->job_t0, s->job_t1));
  return DEFER_OK;
}

int defer_stage_mark(defer_stage_t s, uint64_t seq, int slot) {
  DEFER_CHECK(s && (slot == 0 || slot == 1), "mark: bad arguments");
  DEFER_TRY(set_device(s));
  Mark& m = s->marks[slot];
  if (!m.ev) DEFER_CUDA(cudaEventCreate(&m.ev));
  DEFER_CUDA(cudaEventRecord(m.ev, s->lanes[seq % s->cfg.depth].stream));
  m.recorded = true;
  return DEFER_OK;
}

int defer_stage_mark_elapsed(defer_stage_t s, float* ms) {
  DEFER_CHECK(s && ms, "mark_elapsed: null");
  DEFER_CHECK(s->marks[0].recorded && s->marks[1].recorded, "mark_elapsed: both marks must have been recorded");
  DEFER_TRY(set_device(s));
  DEFER_CUDA(cudaEventSynchronize(s->marks[0].ev));
  DEFER_CUDA(cudaEventSynchronize(s->marks[1].ev));
  DEFER_CUDA(cudaEventElapsedTime(ms, s->marks[0].ev, s->marks[1].ev));
  return DEFER_OK;
}

// ------------------------------------------------------------------------------------------ introspection
int defer_stage_num_kernels(defer_stage_t s, int* per_step) {
  DEFER_CHECK(s && per_step, "num_kernels: null");
  int n = 0;
  for (size_t i = 0; i < s->ops.size(); ++i) {
    auto& op = s->ops[i];
    const int g = s->op_group.empty() ? -1 : s->op_group[i];
    if (g >= 0 && (int)i != s->groups[g].first) continue;   // one launch per megakernel group
    bool is_memcpy = op.d.kind == DEFER_OP_COPY && s->bufs[op.d.in0].elem == DEFER_BUF_F32 && s->bufs[op.d.out].elem == DEFER_BUF_F32;
    if (!is_memcpy) n += op.n_kernels;
  }
  if (s->has_prod) n += 2;  // wait-ready + signal-free
  if (s->has_cons) n += 2;  // wait-free + signal-ready
  *per_step = n;
  return DEFER_OK;
}

int defer_stage_read_buffer(defer_stage_t s, int lane, int buf_id, float* host_out, uint64_t n_floats) {
  DEFER_CHECK(s && host_out && lane >= 0 && lane < s->cfg.depth && buf_id >= 0 && buf_id < (int)s->bufs.size(),
              "read_buffer: bad arguments");
  const Buf& b = s->bufs[buf_id];
  DEFER_CHECK(n_floats == b.elems, "read_buffer: buffer has %zu elements, caller asked %llu", b.elems,
              (unsigned long long)n_floats);
  DEFER_TRY(set_device(s));
  void* src = s->lanes[lane].buf[buf_id];
  DEFER_CHECK(src, "read_buffer: buffer %d is not bound yet", buf_id);
  for (size_t i = 0; i < s->ops.size(); ++i) {
    const OpRt& op = s->ops[i];
    if (op.d.out != buf_id) continue;
    DEFER_CHECK(!(op.d.kind == DEFER_OP_PREPROCESS && op.folded_into >= 0),
                "read_buffer: buffer %d is never written: op %zu (preprocess) is folded into op %d (%s)", buf_id, i,
                op.folded_into, op.folded_into >= 0 ? s->ops[op.folded_into].kname.c_str() : "");
    DEFER_CHECK(op.store_out, "read_buffer: buffer %d is never written: op %zu (%s) stores only the output of the affine op %d "
                "folded into it (no other op reads buffer %d; without DEFER_FOLD_AFFINE=1 it is written)", buf_id, i, op.kname.c_str(),
                op.aff_op, buf_id);
  }
  DEFER_CUDA(cudaStreamSynchronize(s->lanes[lane].stream));
  if (b.elem == DEFER_BUF_PNG || b.elem == DEFER_BUF_IMAGE) {   // the first h * w * 3 bytes of each sample's slot
    const size_t per = (size_t)b.h * b.w * b.c, slot = b.bytes / s->cfg.batch;
    std::vector<uint8_t> raw(b.elems);
    DEFER_CUDA(cudaMemcpy2D(raw.data(), per, src, slot, per, s->cfg.batch, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < b.elems; ++i) host_out[i] = (float)raw[i];
    return DEFER_OK;
  }
  if (b.elem == DEFER_BUF_U8 || b.elem == DEFER_BUF_JPEG) {
    std::vector<uint8_t> raw(b.elems);
    DEFER_CUDA(cudaMemcpy(raw.data(), src, b.elems, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < b.elems; ++i) host_out[i] = (float)raw[i];
    return DEFER_OK;
  }
  if (b.elem == DEFER_BUF_F32 || s->cfg.fmt == DEFER_FMT_F32) {
    DEFER_CUDA(cudaMemcpy(host_out, src, b.elems * 4, cudaMemcpyDeviceToHost));
    return DEFER_OK;
  }
  float* tmp = nullptr;
  DEFER_CUDA(cudaMalloc((void**)&tmp, b.elems * 4));
  int rc = launch_decode(s->cfg.fmt, src, tmp, b.elems, 0);
  cudaError_t e = cudaMemcpy(host_out, tmp, b.elems * 4, cudaMemcpyDeviceToHost);
  cudaFree(tmp);
  if (rc != DEFER_OK) return rc;
  DEFER_CUDA(e);
  return DEFER_OK;
}

int defer_stage_stream(defer_stage_t s, int lane, void** stream) {
  DEFER_CHECK(s && stream && lane >= 0 && lane < s->cfg.depth, "stream: bad arguments");
  *stream = (void*)s->lanes[lane].stream;
  return DEFER_OK;
}

int defer_stage_time_op(defer_stage_t s, int op_index, int iters, int flush_l2, float* us_per_launch) {
  DEFER_CHECK(s && us_per_launch && op_index >= 0 && op_index < (int)s->ops.size() && iters >= 1, "time_op: bad arguments");
  DEFER_CHECK(s->finalized, "time_op: finalize first");
  DEFER_TRY(set_device(s));
  Lane& L = s->lanes[0];
  const defer_op_desc& d = s->ops[op_index].d;
  DEFER_CHECK(L.buf[d.out] && L.buf[d.in0], "time_op: op buffers not bound");
  DEFER_CHECK(s->ops[op_index].folded_into < 0, "time_op: op %d launches nothing, it is folded into op %d (%s)", op_index,
              s->ops[op_index].folded_into, s->ops[op_index].folded_into >= 0 ? s->ops[s->ops[op_index].folded_into].kname.c_str() : "");
  if (flush_l2 && !s->flush_buf) {
    s->flush_bytes = 256ull << 20;  // > 126 MB L2
    DEFER_CUDA(cudaMalloc(&s->flush_buf, s->flush_bytes));
  }
  DEFER_CUDA(cudaStreamSynchronize(L.stream));
  for (int i = 0; i < 3; ++i) DEFER_TRY(launch_op(s, 0, op_index, L.stream));  // warm-up
  double total_ms = 0;
  if (flush_l2) {
    for (int i = 0; i < iters; ++i) {
      DEFER_CUDA(cudaMemsetAsync(s->flush_buf, i & 0xff, s->flush_bytes, L.stream));
      DEFER_CUDA(cudaEventRecord(L.t0, L.stream));
      DEFER_TRY(launch_op(s, 0, op_index, L.stream));
      DEFER_CUDA(cudaEventRecord(L.t1, L.stream));
      DEFER_CUDA(cudaEventSynchronize(L.t1));
      float ms = 0;
      DEFER_CUDA(cudaEventElapsedTime(&ms, L.t0, L.t1));
      total_ms += ms;
    }
  } else {
    DEFER_CUDA(cudaEventRecord(L.t0, L.stream));
    for (int i = 0; i < iters; ++i) DEFER_TRY(launch_op(s, 0, op_index, L.stream));
    DEFER_CUDA(cudaEventRecord(L.t1, L.stream));
    DEFER_CUDA(cudaEventSynchronize(L.t1));
    float ms = 0;
    DEFER_CUDA(cudaEventElapsedTime(&ms, L.t0, L.t1));
    total_ms = ms;
  }
  *us_per_launch = (float)(total_ms * 1000.0 / iters);
  return DEFER_OK;
}

int defer_stage_op_info(defer_stage_t s, int op_index, double* alg_bytes, double* alg_flops, char* kernel_name,
                        int name_len) {
  DEFER_CHECK(s && op_index >= 0 && op_index < (int)s->ops.size(), "op_info: bad arguments");
  const OpRt& op = s->ops[op_index];
  if (alg_bytes) *alg_bytes = op.alg_bytes;
  if (alg_flops) *alg_flops = op.alg_flops;
  if (kernel_name && name_len > 0) {
    strncpy(kernel_name, op.kname.c_str(), name_len - 1);
    kernel_name[name_len - 1] = 0;
  }
  return DEFER_OK;
}

// ------------------------------------------------------------------------------------------ host memory
int defer_host_alloc(void** ptr, uint64_t nbytes) {
  DEFER_CHECK(ptr && nbytes, "host_alloc: bad arguments");
  DEFER_CUDA(cudaMallocHost(ptr, nbytes));
  return DEFER_OK;
}
int defer_host_free(void* ptr) {
  if (ptr) DEFER_CUDA(cudaFreeHost(ptr));
  return DEFER_OK;
}
int defer_host_register(void* ptr, uint64_t nbytes) {
  DEFER_CHECK(ptr && nbytes, "host_register: bad arguments");
  DEFER_CUDA(cudaHostRegister(ptr, nbytes, cudaHostRegisterPortable));
  return DEFER_OK;
}
int defer_host_unregister(void* ptr) {
  if (ptr) DEFER_CUDA(cudaHostUnregister(ptr));
  return DEFER_OK;
}

}  // extern "C"
