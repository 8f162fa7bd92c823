/* defer_b200.h - C-ABI of libdefer_b200.so: the stage operator behind DEFER's node loop.
 *
 * Drop-in boundary (SURVEY.md 8b).  The reference's compute node does, per stage,
 *     part = model_from_json(json); part.set_weights(ws)      (src/node.py:31,34)
 *     out  = part.predict(inpt)                                (src/node.py:105-106)
 *     socket_send(lz4(zfp(out)), next_node)                    (src/node.py:107-108)
 * and the dispatcher feeds / drains the chain (src/dispatcher.py:85-105).  This library replaces
 * exactly that: a *stage* is a fused-op plan + weights resident in HBM on one H100; its forward
 * pass is hand-written sm_90a kernels captured in a CUDA graph per in-flight lane; the hop is a
 * copy-engine transfer (or, optionally, the last kernel's own stores) of the stage output into the
 * next stage's input slot over NVLink (peer or CUDA-IPC mapped) followed by a release flag - no host
 * round trip, no codec (the reference codec is lossless, src/node.py:76-79, so a raw copy is
 * bit-equivalent).  Queue items stay single samples; a stage built with batch = G x item-batch runs
 * G in-flight items per launch (defer_stage_submit_part / _parts).
 *
 * Conventions: every entry point is extern "C", returns 0 on success and a negative defer_status
 * on failure; defer_last_error() gives a thread-local message.  No exception, torch type or C++
 * type crosses the boundary: plain pointers, sizes and POD structs only.  A stage handle is used
 * by one host thread at a time; different stages are independent.
 */
#ifndef DEFER_B200_H_
#define DEFER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DEFER_ABI_VERSION 2

#if defined(DEFER_BUILD)
#define DEFER_API __attribute__((visibility("default")))
#else
#define DEFER_API
#endif

typedef enum defer_status {
  DEFER_OK = 0,
  DEFER_ERR_INVALID = -1,   /* bad argument / unsupported plan */
  DEFER_ERR_CUDA = -2,      /* CUDA runtime or driver error (message has the CUDA string) */
  DEFER_ERR_TIMEOUT = -3,   /* a device-side flag wait gave up (peer stage dead?) */
  DEFER_ERR_STATE = -4      /* call sequence error (e.g. step before link) */
} defer_status;

/* Activation storage format inside a stage and across hops. */
typedef enum defer_fmt {
  DEFER_FMT_F32 = 0,     /* IEEE fp32, SIMT FFMA contractions (exact-order fp32)                       */
  DEFER_FMT_BF16X2 = 1,  /* fp32 carried as two bf16 planes (hi + lo, 4 B/elem): wgmma bf16x3 MMAs,    */
                         /* fp32 accumulate - ~2^-16 relative per layer, meets the 1e-3 fp32 parity bar */
  DEFER_FMT_BF16 = 2     /* one bf16 plane, wgmma bf16 MMA, fp32   accumulate (the bf16 configs)       */
} defer_fmt;

typedef enum defer_op_kind {
  DEFER_OP_CONV = 1,     /* [zero-pad +] conv + per-channel scale/shift (bias+BN folded) [+ residual] [+ relu] */
  DEFER_OP_MAXPOOL = 2,  /* [zero-pad +] max-pool, 'valid'                                                    */
  DEFER_OP_GAP = 3,      /* global average pool  (H,W,C) -> (C)                                               */
  DEFER_OP_DENSE = 4,    /* x @ W + b [+ relu]   (softmax is its own op)                                      */
  DEFER_OP_SOFTMAX = 5,  /* row softmax over C                                                                */
  DEFER_OP_AFFINE = 6,   /* standalone BN: per-channel scale/shift [+ relu]                                   */
  DEFER_OP_RELU = 7,     /* standalone Activation('relu')                                                     */
  DEFER_OP_ADD = 8,      /* standalone Add of two tensors [+ relu]                                            */
  DEFER_OP_PAD = 9,      /* standalone ZeroPadding2D                                                          */
  DEFER_OP_COPY = 10,    /* identity / Flatten / format cast                                                  */
  DEFER_OP_PREPROCESS = 11, /* Keras preprocess_input: in0 = U8 image (c == 3), out = F32 of the same shape;    */
                         /* `mode` DEFER_PRE_CAFFE: w_shift = 3 fp32 values in output-channel order,            */
                         /*   y[..., c] = float(x[..., 2 - c]) + shift[c]  (RGB -> BGR, minus the ImageNet mean)  */
                         /* `mode` DEFER_PRE_TF: no weights, y = float(x) / 127.5 - 1 in fp32 (ResNet V2)       */
  DEFER_OP_RESIZE = 12,  /* Keras load_img(target_size=...) resize, one axis of Pillow's 8-bit resampling:       */
                         /*   in0 = U8 (h_in, w_in, 3), out = U8 (h_out, w_out, 3), exactly one of h / w differs  */
                         /*   (that is the axis; `mode` 0).  Weights are int32 tables of that axis:               */
                         /*   w_scale  = [out_len, 2] (first, count): output i reads source [first, first + count) */
                         /*   w_kernel = [out_len, kw] fixed-point taps, 22 fractional bits;  kw = ksize          */
                         /*   y[i] = clamp((2^21 + sum_{k < count} x[first + k] * tap[k]) >> 22, 0, 255) per     */
                         /*   channel; 0 <= first, 1 <= count <= kw, first + count <= in_len (checked at create)  */
                         /* `mode` DEFER_RESIZE_W / _H: the same on the named axis, which may keep its length    */
                         /* `mode` DEFER_RESIZE_SAMPLE_W / _H: images of mixed sizes, tables per sample (below)   */
  DEFER_OP_JPEG_DECODE = 13, /* baseline JPEG files -> images (below): in0 = the stage input, a DEFER_BUF_JPEG (H, W, 3)   */
                         /*   slot per sample; out = U8 (H, W, 3), each image packed (h, w, 3) at the start of its sample;  */
                         /*   read by the DEFER_RESIZE_SAMPLE_W op.  No weights, mode 0.                                     */
  DEFER_OP_PNG_DECODE = 14, /* non-interlaced PNG files -> images (below): as DEFER_OP_JPEG_DECODE, from a DEFER_BUF_PNG */
                         /*   (H, W, 3) input of DEFER_PNG_SLOT_BYTES(H, W) bytes per sample                                 */
  DEFER_OP_IMAGE_DECODE = 15 /* JPEG or PNG files, each sample its own (below): as DEFER_OP_PNG_DECODE, from a           */
                         /*   DEFER_BUF_IMAGE (H, W, 3) input of DEFER_PNG_SLOT_BYTES(H, W) bytes per sample                 */
} defer_op_kind;

/* defer_op_desc.mode of a DEFER_OP_RESIZE op.  0: the fixed-size resize above (one image size per stage).
 * The two per-sample modes come as a pair and take images of any size up to the stage input (H, W):
 *   DEFER_RESIZE_SAMPLE_W  in0 = the stage input, U8 (H, W, 3)  ->  out U8 (H, W_out, 3)      kw = kw_w
 *   DEFER_RESIZE_SAMPLE_H  in0 = that output, U8 (H, W_out, 3)  ->  out U8 (H_out, W_out, 3)  kw = kw_h
 * They have no weights.  Each sample of a microbatch carries its own int32 table block, written next to its input slot
 * by defer_stage_submit_frames:
 *   [h_in, w_in,  width axis: (first, count) [W_out, 2], taps [W_out, kw_w],
 *                 height axis: (first, count) [H_out, 2], taps [H_out, kw_h]]          (taps zero past count)
 * with 1 <= h_in <= H, 1 <= w_in <= W; the image is packed as (h_in, w_in, 3) at the start of its slot.  An axis whose
 * length equals the target has the identity table (first = i, count 1, tap 2^22).  The arithmetic is mode 0's.  The
 * kernel clamps h_in / w_in, first and count into the slot, so no block content can make it read outside the slot, and
 * the blocks are zeroed at create (a never-written sample reads as a 1x1 image of weight 0).  Both ops are always
 * planned, even when an axis of the bound already equals the target, as the axis cannot be told from the shapes then. */
#define DEFER_RESIZE_SAMPLE_W 1
#define DEFER_RESIZE_SAMPLE_H 2
/* Modes W / H: mode 0's fixed tables on the named axis, the other axis keeping its length.  The named axis may keep its
 * length too: Keras' load_img(keep_aspect_ratio=True) resamples an axis of the target's length when its crop box does
 * not cover it (Pillow's resize with box=), which mode 0 cannot tell from the shapes. */
#define DEFER_RESIZE_W 4
#define DEFER_RESIZE_H 5

/* DEFER_OP_JPEG_DECODE decodes each sample's JPEG file on the GPU, bit for bit as libjpeg-turbo 3.1 does through Pillow
 * (defer_b200/jpeg.py restates it).  It is planned before the DEFER_RESIZE_SAMPLE_W / _H pair, whose table blocks keep
 * their layout.  The sample's file sits at the start of its H * W * 3-byte slot; its int32 block, written next to the
 * slots by defer_stage_submit_jpegs after the resize blocks, is DEFER_JPEG_BLOCK_INTS values:
 *   [0] h  [1] w  [2] components (1 | 3)  [3] luma h-sampling  [4] luma v-sampling (1x1, 2x1 or 2x2; chroma 1x1)
 *   [5] restart interval in MCUs (0 = none)  [6] entropy-data offset in the file  [7] its length (up to EOI)
 *   [8] MCUs across  [9] MCUs down  [10] scans of a progressive file (0: baseline)  [11] Huffman tables in its pool
 *   [12..15] 0
 *   [16 + 64 c ...]  quantisation table of component c, natural order (c < 3)
 *   [16 + 192 + t * DEFER_JPEG_HUFF_INTS ...]  Huffman table t = DC of component 0, 1, 2, then AC of component 0, 1, 2:
 *        lookahead[2^DEFER_JPEG_LOOKAHEAD] (code length << 8 | symbol for codes of <= LOOKAHEAD bits, 0 otherwise),
 *        maxcode[17] (largest code of each length, -1 if none), valoff[17] (symbol index - code), symbols[256]
 * A progressive file (SOF2) leaves those six tables zero; its block goes on with
 *   [DEFER_JPEG_SCAN_OFF + s * DEFER_JPEG_SCAN_INTS ...]  scan s < [10], in file order: components in the scan (all, or
 *        1), their frame indices [3], Ss, Se, Ah, Al, restart interval (MCUs, or blocks of a one-component scan),
 *        entropy-data offset in the file and length, pool index of each component's DC table [3] (DC first scans),
 *        pool index of the AC table (AC scans), 0
 *   [DEFER_JPEG_POOL_OFF + t * DEFER_JPEG_HUFF_INTS ...]  Huffman table t < [11] of the pool, in the layout above
 * A baseline file uses DEFER_JPEG_BASE_INTS values of its block, a progressive one DEFER_JPEG_POOL_OFF + [11] *
 * DEFER_JPEG_HUFF_INTS; only that prefix is copied and read.  A progressive file decodes scan by scan on the same CTA:
 * DC and AC first scans by self-synchronisation, DC refinements one thread per block, AC refinements sequentially, one
 * thread per restart interval.
 * The decode never trusts the block: h / w are clamped into the slot, sampling into 4:4:4 / 4:2:2 / 4:2:0, the entropy
 * extent into the slot and every table index into its table, so no block content makes it access memory outside the
 * sample's slot, workspace or image.  The blocks are zeroed at create: a never-written sample decodes to a 1x1 image of
 * value 128.  An invalid Huffman code ends the sample's decode (that block and all later ones are zero; in a progressive
 * file, they get nothing from that scan and no later scan is decoded); the exact rule for corrupt data is
 * defer_b200/jpeg.py's.  Workspace stats: [0] unstuffed bytes, [1] RST markers, [2] subsequences, [3] rounds, [4] the
 * first block whose decode failed, else the block count; a progressive file sums [0..3] over its scans decoded, gives
 * [4] in the failing scan's block order and [5] the scans decoded whole. */
#define DEFER_JPEG_HDR_INTS 16
#define DEFER_JPEG_LOOKAHEAD 9
#define DEFER_JPEG_HUFF_INTS ((1 << DEFER_JPEG_LOOKAHEAD) + 17 + 17 + 256)
/* the baseline part of a block, all a baseline file uses */
#define DEFER_JPEG_BASE_INTS (DEFER_JPEG_HDR_INTS + 3 * 64 + 6 * DEFER_JPEG_HUFF_INTS)
/* a progressive file: at most this many scans and distinct Huffman tables (more are refused by the parser) */
#define DEFER_JPEG_MAX_SCANS 32
#define DEFER_JPEG_MAX_TABLES 32
#define DEFER_JPEG_SCAN_INTS 16
#define DEFER_JPEG_SCAN_OFF DEFER_JPEG_BASE_INTS
#define DEFER_JPEG_POOL_OFF (DEFER_JPEG_SCAN_OFF + DEFER_JPEG_MAX_SCANS * DEFER_JPEG_SCAN_INTS)
#define DEFER_JPEG_BLOCK_INTS (DEFER_JPEG_POOL_OFF + DEFER_JPEG_MAX_TABLES * DEFER_JPEG_HUFF_INTS)
/* bits per subsequence of the self-synchronising Huffman decode */
#define DEFER_JPEG_SUBSEQ_BITS 8192

/* DEFER_OP_PNG_DECODE decodes each sample's PNG file on the GPU, bit for bit as Pillow's convert("RGB") gives it
 * (defer_b200/png.py restates it, with its one defined result for corrupt data).  It is planned before the
 * DEFER_RESIZE_SAMPLE_W / _H pair, exactly where DEFER_OP_JPEG_DECODE is.  The sample's file sits at the start of its
 * DEFER_PNG_SLOT_BYTES(H, W)-byte slot, room for the stored (level 0) encoding of any accepted image up to (H, W); its
 * int32 block, written next to the slots by defer_stage_submit_pngs after the resize blocks, is DEFER_PNG_BLOCK_INTS
 * values:
 *   [0] h  [1] w  [2] colour type (0, 2, 3, 4, 6)  [3] bit depth  [4] bytes per row (without the filter byte)
 *   [5] filter unit (bytes per complete pixel, at least 1)  [6] IDAT chunks  [7] their total payload bytes
 *   [8] PLTE entries  [9..15] 0
 *   [DEFER_PNG_PAL_OFF + i]           palette entry i < 256: r | g << 8 | b << 16, zero past the PLTE length
 *   [DEFER_PNG_IDAT_OFF + 2 k, + 1]   IDAT chunk k < [6]: payload offset in the file, payload length
 * Only the prefix a file uses, DEFER_PNG_IDAT_OFF + 2 * [6] values, is copied and read.  The device gathers the IDAT
 * payloads into one zlib stream, inflates it (stored, fixed and dynamic Huffman blocks), unfilters the scanlines in a
 * wavefront and converts them to RGB as Pillow does for the file's mode and depth.
 * The decode never trusts the block: h / w are clamped into the slot, colour type and depth to a valid pair (from which
 * it derives the row length itself), every IDAT range into the slot and the stream into its workspace, so no block
 * content makes it access memory outside the sample's slot, workspace or image.  The blocks are zeroed at create: a
 * never-written sample decodes to a 1x1 black image.  Corrupt compressed data ends the stream; the scanline bytes not
 * produced are zero, and a filter type above 4 unfilters its row as None (defer_b200/png.py gives the exact rule).
 * Workspace stats: [0] status (0 complete, 1 final block before the end, 2 input exhausted, 3 bad block type or stored
 * length, 4 bad dynamic header, 5 bad code or symbol, 6 distance too far back), [1] scanline bytes produced, [2] rows
 * with an unknown filter type. */
#define DEFER_PNG_HDR_INTS 16
#define DEFER_PNG_PAL_OFF DEFER_PNG_HDR_INTS
#define DEFER_PNG_IDAT_OFF (DEFER_PNG_PAL_OFF + 256)
/* IDAT chunks of one file (more are refused by the parser; libpng writes 8 KiB chunks) */
#define DEFER_PNG_MAX_IDAT 4096
#define DEFER_PNG_BLOCK_INTS (DEFER_PNG_IDAT_OFF + 2 * DEFER_PNG_MAX_IDAT)
/* one sample's file slot: the stored encoding of RGBA at 16 bits, H * (1 + 8 W) scanline bytes, 1/64 more for block and
 * chunk headers, and 64 KiB for the other chunks */
#define DEFER_PNG_SLOT_BYTES(H, W) ((H) * (1 + 8 * (W)) + (H) * (1 + 8 * (W)) / 64 + 65536)

/* DEFER_OP_IMAGE_DECODE decodes a microbatch whose samples are JPEG or PNG files, each told by its block's tag, bit for
 * bit as the two single-format ops do (defer_b200/image.py).  It is planned where DEFER_OP_JPEG_DECODE is.  The sample's
 * file sits at the start of its DEFER_PNG_SLOT_BYTES(H, W)-byte slot (the larger of the two slots; a JPEG file is still
 * at most H * W * 3 bytes, as jpeg_bound_ok needs); its int32 block of DEFER_IMAGE_BLOCK_INTS values is the file's
 * JPEG or PNG block in that format's layout, with the tag in [DEFER_IMAGE_TAG] (both layouts leave it zero, and the
 * single-format ops never read it).  The op runs the three JPEG kernels on the samples tagged DEFER_IMAGE_JPEG, then the
 * three PNG kernels on every other sample: a never-written (zeroed) sample decodes as in a PNG stage, to a 1x1 black
 * image.  The CTAs of the other format's samples exit after reading the tag.  Each sample's workspace is the larger of
 * the two formats' strides, and holds the layout (stats included) of the format that decoded it. */
#define DEFER_IMAGE_TAG 15
#define DEFER_IMAGE_JPEG 1
#define DEFER_IMAGE_PNG 2
#define DEFER_IMAGE_BLOCK_INTS \
  (DEFER_JPEG_BLOCK_INTS > DEFER_PNG_BLOCK_INTS ? DEFER_JPEG_BLOCK_INTS : DEFER_PNG_BLOCK_INTS)

/* defer_op_desc.mode of a DEFER_OP_PREPROCESS op (every other op kind: 0). */
#define DEFER_PRE_CAFFE 0   /* keras_applications imagenet_utils mode='caffe' (ResNet50/101/152, VGG16) */
#define DEFER_PRE_TF    1   /* mode='tf' (ResNet50V2/101V2/152V2): fl32(fl32(x / 127.5) - 1), bit for bit */

#define DEFER_FLAG_RELU      1u   /* apply relu at the end of the op                 */
#define DEFER_FLAG_RESIDUAL  2u   /* CONV: add buffer in1 before the (optional) relu */

/* Buffer element type. */
#define DEFER_BUF_ACT 0   /* stage activation format (defer_fmt of the stage) */
#define DEFER_BUF_F32 1   /* plain fp32 regardless of the stage format (image in, probabilities out) */
#define DEFER_BUF_U8  2   /* uint8 NHWC, 1 B/elem, first stage only: its input buffer or the output of a DEFER_OP_RESIZE; */
                          /* read only by DEFER_OP_RESIZE and DEFER_OP_PREPROCESS                                          */
                          /* (or of a DEFER_OP_JPEG_DECODE, _PNG_DECODE or _IMAGE_DECODE)                                  */
#define DEFER_BUF_JPEG 3  /* bytes of one JPEG file per sample, h * w * c of them: the first stage's input buffer only,   */
                          /* read only by DEFER_OP_JPEG_DECODE                                                             */
#define DEFER_BUF_PNG 4   /* bytes of one PNG file per sample, DEFER_PNG_SLOT_BYTES(h, w) of them (c = 3): the first      */
                          /* stage's input buffer only, read only by DEFER_OP_PNG_DECODE                                   */
#define DEFER_BUF_IMAGE 5 /* bytes of one JPEG or PNG file per sample, DEFER_PNG_SLOT_BYTES(h, w) of them (c = 3): the    */
                          /* first stage's input buffer only, (h, w) within both formats' bounds; read only by             */
                          /* DEFER_OP_IMAGE_DECODE                                                                         */

/* One logical tensor of the plan.  Shapes are per sample, NHWC; vectors use h = w = 1. */
typedef struct defer_buf_desc {
  int32_t h, w, c;
  int32_t elem;            /* DEFER_BUF_ACT | DEFER_BUF_F32 | DEFER_BUF_U8 | DEFER_BUF_JPEG | DEFER_BUF_PNG |
                              DEFER_BUF_IMAGE */
} defer_buf_desc;

/* One fused op of the plan.  Buffer ids index the defer_buf_desc array; weight ids index the
 * weight-pointer array given to defer_stage_create (-1 = absent). */
typedef struct defer_op_desc {
  int32_t kind;            /* defer_op_kind */
  int32_t in0, in1, out;   /* buffer ids; in1 = residual / second addend, -1 if unused */
  int32_t kh, kw, sh, sw;  /* CONV / MAXPOOL window and stride */
  int32_t pad_t, pad_l, pad_b, pad_r; /* explicit zero padding applied to in0 (fused ZeroPadding2D / 'same') */
  uint32_t flags;          /* DEFER_FLAG_* */
  int32_t w_kernel;        /* CONV: fp32 HWIO kernel;  DENSE: fp32 (in,out) kernel;  RESIZE: int32 taps */
  int32_t w_scale;         /* CONV / AFFINE: fp32 per-channel scale (NULL id -1 = ones);  RESIZE: int32 (first, count) */
  int32_t w_shift;         /* CONV / AFFINE / PREPROCESS: fp32 per-channel shift;  DENSE: bias */
  int32_t mode;            /* PREPROCESS: DEFER_PRE_*;  RESIZE: 0 | DEFER_RESIZE_SAMPLE_*;  every other kind: 0 */
} defer_op_desc;

typedef struct defer_stage_config {
  int32_t abi_version;     /* DEFER_ABI_VERSION */
  int32_t device;          /* CUDA ordinal (reference: a node IP, src/dispatcher.py:45-55) */
  int32_t fmt;             /* defer_fmt */
  int32_t batch;           /* samples per microbatch (reference: 1, test/test.py:22) */
  int32_t depth;           /* in-flight microbatches = input slots = lanes (>= 1) */
  int32_t input_buf;       /* buffer id of the stage input  */
  int32_t output_buf;      /* buffer id of the stage output */
  int32_t is_first;        /* 1: input arrives from host via defer_stage_submit */
  int32_t is_last;         /* 1: output is read back by defer_stage_result */
  int32_t conv_backend;    /* 0 auto, 1 SIMT only, 2 wgmma where eligible (error if fmt == F32) */
  int32_t use_graph;       /* 1: capture each lane's chain into a CUDA graph (default), 0: eager launches */
  int32_t wait_timeout_ms; /* device-side flag wait budget; 0 = default (4000 ms) */
} defer_stage_config;

typedef struct defer_stage_s* defer_stage_t;

/* Size in bytes of the opaque link token produced by defer_stage_export_link. */
#define DEFER_LINK_TOKEN_BYTES 256

/* ---- library ------------------------------------------------------------------------------ */
DEFER_API const char* defer_last_error(void);
DEFER_API int defer_abi_version(void);
DEFER_API int defer_device_count(int* count);
/* name (<=255 chars), SM count, compute capability major*10+minor, total HBM bytes */
DEFER_API int defer_device_info(int device, char* name, int name_len, int* sm_count, int* cc, uint64_t* hbm_bytes);

/* ---- stage life cycle  (replaces model_from_json + set_weights, src/node.py:31-38) ---------- */
/* weights: host pointers to fp32 arrays (int32 for the tables of DEFER_OP_RESIZE), copied; the caller keeps ownership
 * of host memory. */
DEFER_API int defer_stage_create(const defer_stage_config* cfg,
                       const defer_buf_desc* bufs, int n_bufs,
                       const defer_op_desc* ops, int n_ops,
                       const void* const* weight_ptrs, const uint64_t* weight_nbytes, int n_weights,
                       defer_stage_t* out);
DEFER_API int defer_stage_destroy(defer_stage_t s);
/* Human-readable plan / kernel choice dump (replaces plot_model, src/node.py:39). */
DEFER_API int defer_stage_describe(defer_stage_t s, char* buf, size_t buf_len);
/* bytes of one microbatch entering / leaving the stage (hop payload) */
DEFER_API int defer_stage_io_bytes(defer_stage_t s, uint64_t* in_bytes, uint64_t* out_bytes);

/* ---- wiring the chain  (replaces next-hop hand-off, src/dispatcher.py:51-55,63) ------------- */
/* Same process: enable peer access both ways and hand prod the consumer's slots + flags. */
DEFER_API int defer_stage_link(defer_stage_t prod, defer_stage_t cons);
/* Other process (one rank per GPU): the consumer exports a token, the producer imports it, and
 * vice versa for the back-pressure flags.  role: 0 = "my input side" (give to my producer),
 * 1 = "my output side" (give to my consumer). */
DEFER_API int defer_stage_export_link(defer_stage_t s, int role, void* token /* DEFER_LINK_TOKEN_BYTES */);
DEFER_API int defer_stage_import_link(defer_stage_t s, int role, const void* token);
/* Drop the mappings of the neighbours' arenas (CUDA-IPC close).  In a multi-process pipeline every rank
 * calls this, then all ranks synchronise, then each destroys its stage - so no arena is freed while a
 * neighbour still maps it.  The stage cannot step afterwards. */
DEFER_API int defer_stage_unlink(defer_stage_t s);
/* Finish wiring: builds the per-lane CUDA graphs.  Must be called once after linking (also for
 * a single-stage pipeline). */
DEFER_API int defer_stage_finalize(defer_stage_t s);

/* ---- steady state  (replaces the recv -> predict -> send loop, src/node.py:88-91,103-108) --- */
/* First stage only: enqueue the H2D copy of microbatch `seq` from host memory (pinned => async). */
DEFER_API int defer_stage_submit(defer_stage_t s, uint64_t seq, const void* host_in, uint64_t nbytes);
/* First stage only, coalesced ingress: the reference's queue items are single samples (test/test.py:22,47-49); a stage
 * built with batch = G x item-batch runs G in-flight items per launch.  Copies `count` consecutive samples of
 * microbatch `seq`, starting at sample `index`, from host memory (nbytes = count x bytes of one sample). */
DEFER_API int defer_stage_submit_part(defer_stage_t s, uint64_t seq, int index, int count, const void* host_in, uint64_t nbytes);
/* The same for a run of queue items in ONE call (the dispatcher's feeder gathers the items of a group, then ships them):
 * item i (samples_per_item samples, nbytes_per_item bytes at host_ptrs[i]) goes to samples
 * [first_index + i * samples_per_item, ...). */
DEFER_API int defer_stage_submit_parts(defer_stage_t s, uint64_t seq, int first_index, int n_items, int samples_per_item,
                             const void* const* host_ptrs, uint64_t nbytes_per_item);
/* First stage with a DEFER_RESIZE_SAMPLE_W / _H pair, images of mixed sizes: image i (hw[i] = (h, w), 1 <= h <= H,
 * 1 <= w <= W of the stage input; h * w * 3 contiguous bytes at images[i]) goes to the start of sample slot
 * first_index + i, and its table block (tables: n blocks, table_bytes = n x block bytes; header (h, w) equal to hw[i])
 * next to the slots.  Only the images' own bytes are copied.  Everything is checked before anything is copied
 * (DEFER_ERR_INVALID, nothing copied).  The copies go on the lane's stream; memory as for defer_stage_submit.
 * defer_stage_submit / _part / _parts refuse such a stage. */
DEFER_API int defer_stage_submit_frames(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* images,
                              const int32_t* hw /* [n][2] */, const int32_t* tables, uint64_t table_bytes);
/* First stage with a DEFER_OP_JPEG_DECODE op: file i (nbytes[i] bytes at data[i], at most H * W * 3) goes to the start of
 * sample slot first_index + i.  blocks holds, per file, its resize table block followed by its JPEG block
 * (block_bytes = n x (resize block + DEFER_JPEG_BLOCK_INTS) x 4); the resize header (h, w) must equal the JPEG block's,
 * with 1 <= h <= H, 1 <= w <= W, and the entropy extent must lie inside the file.  Everything is checked before anything
 * is copied (DEFER_ERR_INVALID, nothing copied); then only each file's own bytes and the blocks are copied, on the lane's
 * stream.  defer_stage_submit / _part / _parts / _frames refuse such a stage. */
DEFER_API int defer_stage_submit_jpegs(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                             const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes);
/* First stage with a DEFER_OP_PNG_DECODE op: the same contract as defer_stage_submit_jpegs, with PNG files of at most
 * DEFER_PNG_SLOT_BYTES(H, W) bytes and DEFER_PNG_BLOCK_INTS-value blocks; each block's IDAT count must be at most
 * DEFER_PNG_MAX_IDAT, its ranges inside the file, and its row length and filter unit those of its size, colour type and
 * depth.  Only the block prefix a file uses is copied.  defer_stage_submit / _part / _parts / _frames / _jpegs refuse
 * such a stage. */
DEFER_API int defer_stage_submit_pngs(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                             const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes);
/* First stage with a DEFER_OP_IMAGE_DECODE op: the same contract, with JPEG or PNG files and DEFER_IMAGE_BLOCK_INTS-value
 * blocks, each tagged DEFER_IMAGE_JPEG or DEFER_IMAGE_PNG in [DEFER_IMAGE_TAG].  Each file meets the checks of
 * defer_stage_submit_jpegs or _pngs for its tag; a JPEG file is at most H * W * 3 bytes, a PNG file at most
 * DEFER_PNG_SLOT_BYTES(H, W).  Only the block prefix a file uses is copied.  Every other submit call refuses such a
 * stage. */
DEFER_API int defer_stage_submit_images(defer_stage_t s, uint64_t seq, int first_index, int n, const void* const* data,
                              const uint64_t* nbytes, const int32_t* blocks, uint64_t block_bytes);
/* Enqueue microbatch `seq` on lane seq % depth: wait-input -> kernel chain -> hop -> flags. Async. */
DEFER_API int defer_stage_step(defer_stage_t s, uint64_t seq);
/* Last stage only: block until microbatch `seq` is complete and copy its fp32 output to host.  A lane keeps only the output
 * of the latest microbatch stepped on it, so at most `depth` microbatches may be stepped from `seq` on before its result is
 * collected: DEFER_ERR_STATE if lane seq % depth has run a later microbatch since, or never ran `seq`. */
DEFER_API int defer_stage_result(defer_stage_t s, uint64_t seq, void* host_out, uint64_t nbytes);
/* Convenience for single-stage use: submit + step + result. */
DEFER_API int defer_stage_predict(defer_stage_t s, const void* host_in, uint64_t in_bytes, void* host_out, uint64_t out_bytes);
DEFER_API int defer_stage_sync(defer_stage_t s);
/* Sticky device-side status: 0 ok, DEFER_ERR_TIMEOUT if a flag wait expired. */
DEFER_API int defer_stage_status(defer_stage_t s);
/* Device time of the last completed step on `lane` in microseconds (CUDA events on the lane's stream). */
DEFER_API int defer_stage_last_step_us(defer_stage_t s, int lane, float* us);

/* Whole-job device timing across all lanes (CUDA events, no host clock): start records T0 on lane 0's
 * stream (call it when the stage is idle, right before the first step of the timed region); stop makes
 * lane 0 wait for every lane, records T1, synchronises and returns T1 - T0 in milliseconds. */
DEFER_API int defer_stage_timer_start(defer_stage_t s);
DEFER_API int defer_stage_timer_stop(defer_stage_t s, float* ms);

/* Steady-state timing without draining the pipeline (the reference protocol counts results inside a window while the
 * chain stays flooded, test/test.py:25-36): call mark(seq, slot) right after step(seq); it records a CUDA event behind
 * that microbatch on its lane.  mark_elapsed = device time from the completion of the slot-0 microbatch to the
 * completion of the slot-1 microbatch. */
DEFER_API int defer_stage_mark(defer_stage_t s, uint64_t seq, int slot /* 0 | 1 */);
DEFER_API int defer_stage_mark_elapsed(defer_stage_t s, float* ms);

/* ---- introspection for tests and benches --------------------------------------------------- */
DEFER_API int defer_stage_num_kernels(defer_stage_t s, int* per_step);           /* kernel launches per step */
/* copy any plan buffer of `lane` to host as fp32 NHWC (decodes the stage format; a U8 buffer reads as its values
 * 0..255).  Fails for the F32 image of a PREPROCESS op folded into the stem conv: that buffer is never written. */
DEFER_API int defer_stage_read_buffer(defer_stage_t s, int lane, int buf_id, float* host_out, uint64_t n_floats);
/* stream / event handles for external timing (cudaStream_t as void*) */
DEFER_API int defer_stage_stream(defer_stage_t s, int lane, void** stream);
/* time `iters` back-to-back launches of op `op_index` alone on lane 0 (CUDA events); microseconds per launch */
DEFER_API int defer_stage_time_op(defer_stage_t s, int op_index, int iters, int flush_l2, float* us_per_launch);
/* algorithmic bytes and flops of op `op_index` (SURVEY.md 8d formula) and its kernel name */
DEFER_API int defer_stage_op_info(defer_stage_t s, int op_index, double* alg_bytes, double* alg_flops,
                        char* kernel_name, int name_len);

/* ---- host memory helpers -------------------------------------------------------------------- */
DEFER_API int defer_host_alloc(void** ptr, uint64_t nbytes);     /* pinned */
DEFER_API int defer_host_free(void* ptr);
DEFER_API int defer_host_register(void* ptr, uint64_t nbytes);   /* page-lock caller memory in place */
DEFER_API int defer_host_unregister(void* ptr);

/* ---- per-kernel entry points (raw device pointers, e.g. torch.Tensor.data_ptr(); NHWC) ------ */
/* Each runs ONE kernel on `stream` (cudaStream_t as void*, NULL = default) so it can be parity-
 * tested and profiled alone.  Activation tensors are in `fmt`; planes of BF16X2 are
 * [hi | lo], lo at element offset n*h*w*c. Weights: fp32 HWIO + fp32 scale/shift (may be NULL). */
/* backend: 1 SIMT FFMA | 2 wgmma, one tile per CTA (conv_umma_kernel) | 3 persistent grid, 64-wide N tiles (conv_stream_kernel) |
 *          4 / 5 streaming persistent kernel (conv_stream_kernel) with 64- / 128-wide N tiles |
 *          6 / 7 the same, planned for an output in a peer GPU's slot */
DEFER_API int defer_k_conv(int fmt, int backend,
                 const void* x, int x_is_f32, const float* w_hwio, const float* scale, const float* shift,
                 const void* residual, void* y,
                 int n, int h, int w, int cin, int cout, int kh, int kw, int sh, int sw,
                 int pad_t, int pad_l, int pad_b, int pad_r, uint32_t flags, void* stream);
DEFER_API int defer_k_maxpool(int fmt, const void* x, void* y, int n, int h, int w, int c,
                    int ph, int pw, int sh, int sw, int pad_t, int pad_l, int pad_b, int pad_r, void* stream);
DEFER_API int defer_k_gap(int fmt, const void* x, void* y, int n, int h, int w, int c, void* stream);
DEFER_API int defer_k_dense(int fmt, const void* x, const float* w_io, const float* bias, void* y, int y_is_f32,
                  int n, int in_features, int units, uint32_t flags, void* stream);
DEFER_API int defer_k_softmax(const float* x, float* y, int n, int c, void* stream);
DEFER_API int defer_k_eltwise(int fmt, int kind /* AFFINE | RELU | ADD */, const void* a, const void* b,
                    const float* scale, const float* shift, void* y, int n, int h, int w, int c,
                    uint32_t flags, void* stream);
/* fp32 <-> stage-format conversion of a whole tensor (device pointers) */
DEFER_API int defer_k_encode(int fmt, const float* x_f32, void* y_act, uint64_t n_elems, void* stream);
DEFER_API int defer_k_decode(int fmt, const void* x_act, float* y_f32, uint64_t n_elems, void* stream);
/* Keras caffe-mode preprocess_input (DEFER_OP_PREPROCESS): uint8 NHWC image (c == 3) -> fp32,
 * y[..., c] = float(x[..., 2 - c]) + shift[c]; shift: 3 fp32 values on the device */
DEFER_API int defer_k_preprocess(const uint8_t* x, const float* shift, float* y, int n, int h, int w, int c, void* stream);
/* Keras tf-mode preprocess_input (DEFER_OP_PREPROCESS, DEFER_PRE_TF): uint8 NHWC image (c == 3) -> fp32,
 * y = fl32(fl32(float(x) / 127.5) - 1), channels in place */
DEFER_API int defer_k_preprocess_tf(const uint8_t* x, float* y, int n, int h, int w, int c, void* stream);
/* One pass of DEFER_OP_RESIZE: uint8 NHWC (n, h_in, w_in, c == 3) -> (n, h_out, w_out, 3), exactly one axis changing.
 * bounds = int32 [out_len, 2] (first, count) and taps = int32 [out_len, ksize] on the device (not validated here). */
DEFER_API int defer_k_resize(const uint8_t* x, uint8_t* y, const int32_t* bounds, const int32_t* taps, int ksize, int n,
                             int h_in, int w_in, int h_out, int w_out, int c, void* stream);

/* One pass of a DEFER_RESIZE_SAMPLE_W / _H pair (pass = that mode) over n samples: SAMPLE_W reads x = (n, H, W, 3) slots
 * and writes y = (n, H, W_out, 3); SAMPLE_H reads x = (n, H, W_out, 3) and writes y = (n, H_out, W_out, 3).  tables = n
 * int32 blocks of the layout above (kw_w, kw_h taps), on the device, 4-byte aligned; c must be 3. */
DEFER_API int defer_k_resize_frames(int pass, const uint8_t* x, uint8_t* y, const int32_t* tables, int n, int H, int W,
                                    int H_out, int W_out, int kw_w, int kw_h, int c, void* stream);

/* The whole DEFER_OP_JPEG_DECODE of n samples: files = n slots of H * W * 3 bytes, blocks = n JPEG blocks (layout above,
 * 4-byte aligned), y = n U8 (H, W, 3) images; workspace of defer_k_jpeg_workspace bytes, 256-byte aligned, caller-owned.
 * Per sample (sample_stride apart) the workspace holds, from coef_off, the final quantised coefficients as int16 [blocks,
 * 64] in stream order and natural coefficient order, and from plane_off the MCU-padded component planes (uint8, one after
 * the other, each (8 * blocks down) x (8 * blocks across)).  Its first 5 int32 are the unstuffed entropy bytes, the RST
 * markers found, the subsequences, the synchronisation rounds and the blocks before the first invalid code. */
DEFER_API int defer_k_jpeg_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* coef_off,
                                     uint64_t* plane_off);
DEFER_API int defer_k_jpeg_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace,
                                  uint8_t* y, void* stream);

/* The whole DEFER_OP_PNG_DECODE of n samples: files = n slots of DEFER_PNG_SLOT_BYTES(H, W) bytes, blocks = n PNG blocks
 * (layout above, 4-byte aligned), y = n U8 (H, W, 3) images; workspace of defer_k_png_workspace bytes, 256-byte aligned,
 * caller-owned.  Per sample (sample_stride apart) the workspace holds the three stats above as its first int32 values,
 * and from raw_off the scanlines, h * (1 + bytes per row), unfiltered (each row's filter type byte kept). */
DEFER_API int defer_k_png_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* raw_off);
DEFER_API int defer_k_png_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace,
                                 uint8_t* y, void* stream);

/* The whole DEFER_OP_IMAGE_DECODE of n samples: files = n slots of DEFER_PNG_SLOT_BYTES(H, W) bytes, blocks = n tagged
 * blocks of DEFER_IMAGE_BLOCK_INTS values (4-byte aligned), y = n U8 (H, W, 3) images; workspace of
 * defer_k_image_workspace bytes, 256-byte aligned, caller-owned.  Per sample (sample_stride apart) the workspace holds
 * the layout of the format that decoded it: a JPEG sample's stats, coefficients from coef_off and planes from plane_off
 * as defer_k_jpeg_decode writes them; a PNG sample's stats and scanlines from raw_off as defer_k_png_decode does. */
DEFER_API int defer_k_image_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* coef_off,
                                      uint64_t* plane_off, uint64_t* raw_off);
DEFER_API int defer_k_image_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace,
                                   uint8_t* y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DEFER_B200_H_ */
