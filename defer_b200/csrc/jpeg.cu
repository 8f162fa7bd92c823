// jpeg.cu - DEFER_OP_JPEG_DECODE: baseline and progressive JPEG files decoded on the GPU, bit for bit as libjpeg-turbo 3.1 (through Pillow)
// decodes them, and as defer_b200/jpeg.py restates it.  Three kernels per microbatch, each with a fixed grid sized from the
// slot bound (H, W) and an early exit per sample:
//   jpeg_entropy_kernel  one CTA per sample: unstuff the entropy data, Huffman-decode it by self-synchronisation,
//                        write de-zigzagged int16 coefficients, then the DC prediction as a segmented prefix sum; a
//                        progressive file does this scan by scan (progressive_decode), AC refinements sequentially
//   jpeg_idct_kernel     dequantise + libjpeg's integer ISLOW IDCT, 8 threads per 8x8 block, into MCU-padded planes
//   jpeg_color_kernel    libjpeg-turbo's fancy upsampling (h2v1 / h2v2) + jdcolor.c's fixed-point YCbCr -> RGB, one
//                        thread per pixel, packed (h, w, 3) at the start of the sample's U8 slot
// Nothing here trusts the per-sample block: sizes, sampling, offsets and table entries are clamped, so a stale, zero or
// corrupt block gives wrong pixels, never an access outside the sample's slot or workspace.
#include <climits>

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace defer {

namespace {

constexpr int JT = 512;          // threads of the entropy kernel (one CTA per sample)
constexpr int UNSTUFF_ITEMS = 8; // entropy bytes per thread per unstuff step
constexpr int S_BITS = DEFER_JPEG_SUBSEQ_BITS;
constexpr int LUT = 1 << DEFER_JPEG_LOOKAHEAD;
constexpr int HUFF = DEFER_JPEG_HUFF_INTS;
constexpr int Q_OFF = DEFER_JPEG_HDR_INTS;
constexpr int T_OFF = DEFER_JPEG_HDR_INTS + 3 * 64;

__constant__ int c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Geometry of one sample, derived from its block header and clamped into the slot (H, W).
struct Geom {
  int h, w, ncomp, hs, vs, ri;
  int mcux, mcuy, mcus, bpm, nb0, blocks, nseg;
  int bw[3], bh[3];
  size_t poff[3];
  int off, len;   // entropy data within the file slot
};

__device__ __forceinline__ Geom geom(const int32_t* blk, int H, int W, size_t slot) {
  Geom g;
  g.h = min(max(blk[0], 1), H);
  g.w = min(max(blk[1], 1), W);
  g.ncomp = blk[2] == 3 ? 3 : 1;
  g.hs = g.ncomp == 3 ? min(max(blk[3], 1), 2) : 1;
  g.vs = g.ncomp == 3 ? min(max(blk[4], 1), 2) : 1;
  if (g.vs == 2) g.hs = 2;               // 4:4:0 is refused by the parser; keep a corrupt block inside 4:2:0's bounds
  g.ri = min(max(blk[5], 0), 65535);
  const long long off = min(max((long long)blk[6], 0ll), (long long)slot);
  g.off = (int)off;
  g.len = (int)min(max((long long)blk[7], 0ll), (long long)slot - off);
  g.mcux = (g.w + 8 * g.hs - 1) / (8 * g.hs);
  g.mcuy = (g.h + 8 * g.vs - 1) / (8 * g.vs);
  g.mcus = g.mcux * g.mcuy;
  g.nb0 = g.hs * g.vs;
  g.bpm = g.ncomp == 3 ? g.nb0 + 2 : 1;
  g.blocks = g.mcus * g.bpm;
  g.nseg = g.ri ? (g.mcus + g.ri - 1) / g.ri : 1;
  size_t p = 0;
  for (int c = 0; c < 3; ++c) {
    const bool y = c == 0;
    g.bw[c] = c < g.ncomp ? g.mcux * (y ? g.hs : 1) : 0;
    g.bh[c] = c < g.ncomp ? g.mcuy * (y ? g.vs : 1) : 0;
    g.poff[c] = p;
    p += (size_t)g.bw[c] * g.bh[c] * 64;
  }
  return g;
}

__device__ __forceinline__ int comp_of(const Geom& g, int j) { return j < g.nb0 ? 0 : j - g.nb0 + 1; }

// 16 bits at bit `pos` of buf, MSB first; bytes at or past end_bits / 8 read as zero (end_bits is a byte multiple)
__device__ __forceinline__ uint32_t peek16(const uint8_t* __restrict__ buf, int pos, int end_bits) {
  if (pos >= end_bits) return 0;
  const int i = pos >> 3, nb = end_bits >> 3;
  uint32_t v = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) v = (v << 8) | (i + q < nb ? (uint32_t)buf[i + q] : 0u);
  return (v >> (16 - (pos & 7))) & 0xFFFFu;
}

// symbol of the code at the top of `p` and its length, or -1 for an invalid code (table layout: include/defer_b200.h)
__device__ __forceinline__ int decode_sym(const int* __restrict__ t, uint32_t p, int& len) {
  const int e = t[p >> (16 - DEFER_JPEG_LOOKAHEAD)];
  if (e) {
    len = min(max(e >> 8, 1), 16);
    return e & 255;
  }
  for (int l = DEFER_JPEG_LOOKAHEAD + 1; l <= 16; ++l) {
    const int code = (int)(p >> (16 - l));
    if (code <= t[LUT + l]) {
      len = l;
      return t[LUT + 34 + min(max(code + t[LUT + 17 + l], 0), 255)] & 255;
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

// One symbol (code + extra bits) at coefficient k of a block (0 = DC).  Advances pos and k (k == 64 ends the block) and
// sets z (zigzag index written, -1 for none) and v.  false: invalid code, or an AC run past coefficient 63.
__device__ __forceinline__ bool jstep(const uint8_t* __restrict__ buf, int end_bits, const int* dct, const int* act,
                                      int& pos, int& k, int& z, int& v) {
  const uint32_t p = peek16(buf, pos, end_bits);
  int l;
  if (k == 0) {
    int s = decode_sym(dct, p, l);
    if (s < 0) return false;
    s &= 15;
    pos += l;
    v = s ? extend((int)(peek16(buf, pos, end_bits) >> (16 - s)), s) : 0;
    pos += s;
    k = 1;
    z = 0;
    return true;
  }
  const int sym = decode_sym(act, p, l);
  if (sym < 0) return false;
  pos += l;
  const int r = sym >> 4, s = sym & 15;
  z = -1;
  if (s == 0) {
    if (r != 15) {
      k = 64;
      return true;
    }
    if (k + 16 > 64) return false;
    k += 16;
    return true;
  }
  if (k + r > 63) return false;
  v = extend((int)(peek16(buf, pos, end_bits) >> (16 - s)), s);
  pos += s;
  z = k + r;
  k = z + 1;
  return true;
}

// Decode from state (pos, j << 8 | k) to the first symbol boundary at or past `end`; returns the blocks that start before
// `end`.  An invalid code restarts the decode one bit later at block 0, coefficient 0.  A decoder that started at a guessed
// state meets invalid codes often; if it stopped there, the true state could only reach the subsequences behind it one
// per round.  On the true path an invalid code is a real error: the write pass finds it and cuts the decode there, so
// what this path does after it is never used.
__device__ int sync_run(const uint8_t* __restrict__ buf, int seg_end, int end, const int* tabs, const Geom& g, int& pos,
                        int& jk) {
  int j = jk >> 8, k = jk & 255, count = 0;
  while (pos < end) {
    if (k == 0) ++count;
    const int c = comp_of(g, j);
    const int p0 = pos;
    int z, v;
    if (!jstep(buf, seg_end, tabs + c * HUFF, tabs + (3 + c) * HUFF, pos, k, z, v)) {
      pos = p0 + 1;
      j = k = 0;
      continue;
    }
    if (k >= 64) {
      k = 0;
      j = j + 1 == g.bpm ? 0 : j + 1;
    }
  }
  jk = (j << 8) | k;
  return count;
}

struct SegPair {
  int f;
  unsigned v;
};
struct SegSum {
  __device__ __forceinline__ SegPair operator()(const SegPair& a, const SegPair& b) const {
    return SegPair{a.f | b.f, b.f ? b.v : a.v + b.v};
  }
};

}  // namespace

// Per-sample workspace layout (byte offsets from the sample's base); host and device compute it the same way.
struct JpegWs {
  size_t stats, coef, planes, comp, seg_start, seg_total, sub_base, sub, stride;
  int mcu_cap, blocks_cap, subs_cap;
  size_t slot;      // H * W * 3: the extent clamp of a file, and the image stride
  size_t file;      // the file slot stride (DecodeStrides)
  int block_ints;   // the block stride
  int take;         // which samples (decode_takes)
};
enum { SUB_SEG, SUB_EPOS, SUB_EJK, SUB_XPOS, SUB_XJK, SUB_CNT, SUB_PRE, SUB_PPOS, SUB_PJK, SUB_FIELDS };

__host__ __device__ inline JpegWs jpeg_ws(int H, int W) {
  JpegWs L;
  const int hp = (H + 15) / 16 * 16, wp = (W + 15) / 16 * 16;
  L.slot = (size_t)H * W * 3;
  L.mcu_cap = (hp / 8) * (wp / 8);
  L.blocks_cap = 3 * L.mcu_cap;
  L.subs_cap = (int)((L.slot * 8 + S_BITS - 1) / S_BITS) + L.mcu_cap;
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  size_t o = 0;
  L.stats = o;      o += al(64);
  L.coef = o;       o += al((size_t)L.blocks_cap * 128);
  L.planes = o;     o += al((size_t)L.blocks_cap * 64);
  L.comp = o;       o += al(L.slot + 16);
  L.seg_start = o;  o += al(((size_t)L.mcu_cap + 2) * 4);
  L.seg_total = o;  o += al(((size_t)L.mcu_cap + 1) * 4);
  L.sub_base = o;   o += al(((size_t)L.mcu_cap + 1) * 4);
  L.sub = o;        o += al((size_t)L.subs_cap * SUB_FIELDS * 4);
  L.stride = o;
  L.file = L.slot;
  L.block_ints = DEFER_JPEG_BLOCK_INTS;
  L.take = 0;
  return L;
}

namespace {

using ScanI = cub::BlockScan<int, JT>;
using ScanP = cub::BlockScan<SegPair, JT>;

// Steps 1 and 2 of a scan's decode.  1: unstuff the `len` entropy bytes at src into comp (drop 0x00 / RSTn after 0xFF and
// the 0xFF of RSTn) and record where each of the `nseg` restart intervals starts.  2: seg_start[0..nseg], seg_total = 0,
// sub_base (first subsequence of S_BITS bits of each interval).  T: unstuffed bytes, R: RST markers, nsubs: subsequences.
__device__ __forceinline__ void unstuff_intervals(const uint8_t* __restrict__ src, int len, int nseg, uint8_t* comp,
                                                  int32_t* seg_start, int32_t* seg_total, int32_t* sub_base, int subs_cap,
                                                  typename ScanI::TempStorage& tmp, int& T, int& R, int& nsubs) {
  const int tid = threadIdx.x;
  int out_n = 0, rst_n = 0;
  for (int c0 = 0; c0 < len; c0 += JT * UNSTUFF_ITEMS) {
    const int i0 = c0 + tid * UNSTUFF_ITEMS;
    uint8_t b[UNSTUFF_ITEMS];
    unsigned keep = 0, mark = 0;
    int nk = 0, nr = 0;
#pragma unroll
    for (int q = 0; q < UNSTUFF_ITEMS; ++q) {
      const int i = i0 + q;
      b[q] = 0;
      if (i >= len) continue;
      const int x = src[i], prev = i > 0 ? src[i - 1] : 0, next = i + 1 < len ? src[i + 1] : 0;
      b[q] = (uint8_t)x;
      const bool rst = x >= 0xD0 && x <= 0xD7, m = x == 0xFF && next >= 0xD0 && next <= 0xD7;
      if (!((prev == 0xFF && (x == 0 || rst)) || m)) keep |= 1u << q, ++nk;
      if (m) mark |= 1u << q, ++nr;
    }
    int pre, tot;
    ScanI(tmp).ExclusiveSum(nk | (nr << 16), pre, tot);
    int pos = out_n + (pre & 0xFFFF), r = rst_n + (pre >> 16);
#pragma unroll
    for (int q = 0; q < UNSTUFF_ITEMS; ++q) {
      if (mark >> q & 1) {
        if (r + 1 <= nseg) seg_start[r + 1] = pos;
        ++r;
      }
      if (keep >> q & 1) comp[pos++] = b[q];
    }
    out_n += tot & 0xFFFF;
    rst_n += tot >> 16;
    __syncthreads();
  }
  T = out_n;
  R = rst_n;
  for (int k = tid; k <= nseg; k += JT) {
    if (k == 0) seg_start[0] = 0;
    else if (k > R) seg_start[k] = T;
    if (k < nseg) seg_total[k] = 0;
  }
  __syncthreads();
  nsubs = 0;
  for (int k0 = 0; k0 < nseg; k0 += JT) {
    const int k = k0 + tid;
    const int n_k = k < nseg ? (int)(((long long)(seg_start[k + 1] - seg_start[k]) * 8 + S_BITS - 1) / S_BITS) : 0;
    int pre, tot;
    ScanI(tmp).ExclusiveSum(n_k, pre, tot);
    if (k < nseg) sub_base[k] = nsubs + pre;
    nsubs += tot;
    __syncthreads();
  }
  nsubs = min(nsubs, subs_cap);
}

// ------------------------------------------------------------------------------------------------ progressive files
// A progressive file (block word [10] = its scan count) is decoded scan by scan, in file order, into the same
// stream-order coefficients the baseline path writes.  Each scan's entropy data is unstuffed and cut into restart
// intervals as a baseline scan's.  DC first and AC first scans decode by the same self-synchronisation: the state at a
// symbol boundary is still (bit, block within the unit, k), and an EOB run only adds to the blocks a subsequence owns.
// A DC refinement scan is one raw bit per block, one thread per block.  An AC refinement scan reads a correction bit for
// every coefficient that is already non-zero, so where its bits go depends on each block's history: it decodes
// sequentially, one thread per restart interval.
struct PScan {
  int per, units, nq, nseg, ri;   // blocks per unit (the MCU of an interleaved scan, else 1), units, blocks, intervals
  int comp, ss, se, ah, al;       // comp: the component of a one-component scan
  int off, len;                   // entropy data within the file slot
  int dct[3], act;                // pool indices
  int cw, hc, vc;                 // one-component scans: the component's own grid width and its sampling
};

__device__ __forceinline__ PScan pscan(const int32_t* e, const Geom& g, int ntab, size_t slot) {
  PScan p;
  p.ss = min(max(e[4], 0), 63);
  p.se = p.ss == 0 ? 0 : min(max(e[5], p.ss), 63);
  const bool inter = e[0] > 1 && g.ncomp == 3 && p.ss == 0;
  p.comp = inter ? 0 : min(max(e[1], 0), g.ncomp - 1);
  p.ah = min(max(e[6], 0), 13);
  p.al = min(max(e[7], 0), 13);
  p.ri = min(max(e[8], 0), 65535);
  const long long off = min(max((long long)e[9], 0ll), (long long)slot);
  p.off = (int)off;
  p.len = (int)min(max((long long)e[10], 0ll), (long long)slot - off);
  for (int c = 0; c < 3; ++c) p.dct[c] = min(max(e[11 + c], 0), max(ntab - 1, 0));
  p.act = min(max(e[14], 0), max(ntab - 1, 0));
  p.hc = p.comp == 0 ? g.hs : 1;
  p.vc = p.comp == 0 ? g.vs : 1;
  if (inter || g.ncomp == 1) {
    p.per = inter ? g.bpm : 1;
    p.units = g.mcus;
    p.cw = g.mcux;
  } else {
    p.per = 1;
    p.cw = (g.w * p.hc + 8 * g.hs - 1) / (8 * g.hs);
    p.units = p.cw * ((g.h * p.vc + 8 * g.vs - 1) / (8 * g.vs));
  }
  p.nq = p.units * p.per;
  p.nseg = p.ri ? (p.units + p.ri - 1) / p.ri : 1;
  return p;
}

// stream-order block of block q of the scan, in scan order
__device__ __forceinline__ int scan_block(const Geom& g, const PScan& p, int q) {
  if (p.per > 1 || g.ncomp == 1) return q;
  const int bx = q % p.cw, by = q / p.cw;
  if (p.comp == 0) return ((by / p.vc) * g.mcux + bx / p.hc) * g.bpm + (by % p.vc) * p.hc + bx % p.hc;
  return (by * g.mcux + bx) * g.bpm + g.nb0 + p.comp - 1;
}

// One symbol of a DC first or AC first scan at coefficient k of a block at position j of its unit.  As jstep, and
// eob: the blocks after this one that an EOB run ends too.  k > se ends the block.  false: invalid code, or a run past Se.
__device__ __forceinline__ bool pstep(const uint8_t* __restrict__ buf, int end_bits, const int* tabs, const PScan& p,
                                      const Geom& g, int j, int& pos, int& k, int& z, int& v, int& eob) {
  const uint32_t w = peek16(buf, pos, end_bits);
  int l;
  eob = 0;
  if (p.ss == 0) {
    int s = decode_sym(tabs + (p.per > 1 ? comp_of(g, j) : 0) * HUFF, w, l);
    if (s < 0) return false;
    s &= 15;
    pos += l;
    v = s ? extend((int)(peek16(buf, pos, end_bits) >> (16 - s)), s) : 0;
    pos += s;
    z = 0;
    k = 1;
    return true;
  }
  const int sym = decode_sym(tabs + 3 * HUFF, w, l);
  if (sym < 0) return false;
  pos += l;
  const int r = sym >> 4, s = sym & 15;
  z = -1;
  if (s == 0) {
    if (r == 15) {
      if (k + 16 > p.se + 1) return false;
      k += 16;
      return true;
    }
    eob = r ? (1 << r) - 1 + (int)(peek16(buf, pos, end_bits) >> (16 - r)) : 0;
    pos += r;
    k = p.se + 1;
    return true;
  }
  if (k + r > p.se) return false;
  v = extend((int)(peek16(buf, pos, end_bits) >> (16 - s)), s);
  pos += s;
  z = k + r;
  k = z + 1;
  return true;
}

// sync_run for a DC first or AC first scan (block start: k == Ss); the count includes the blocks of EOB runs
__device__ int psync_run(const uint8_t* __restrict__ buf, int seg_end, int end, const int* tabs, const PScan& p,
                         const Geom& g, int& pos, int& jk) {
  int j = jk >> 8, k = jk & 255, count = 0;
  while (pos < end) {
    if (k == p.ss) ++count;
    const int p0 = pos;
    int z, v, eob;
    if (!pstep(buf, seg_end, tabs, p, g, j, pos, k, z, v, eob)) {
      pos = p0 + 1;
      j = 0;
      k = p.ss;
      continue;
    }
    count += eob;
    if (k > p.se) {
      k = p.ss;
      j = j + 1 == p.per ? 0 : j + 1;
    }
  }
  jk = (j << 8) | k;
  return min(count, g.blocks);
}

__device__ __forceinline__ int getbit(const uint8_t* __restrict__ buf, int pos, int end_bits) {
  return pos < end_bits ? (buf[pos >> 3] >> (7 - (pos & 7))) & 1 : 0;
}

// position of the n-th (from 0) set bit of x; x has more than n set bits
__device__ __forceinline__ int nth_bit(uint64_t x, int n) {
  const unsigned lo = (unsigned)x, c = __popc(lo);
  return n < (int)c ? (int)__fns(lo, 0, n + 1) : 32 + (int)__fns((unsigned)(x >> 32), 0, n - c + 1);
}

// one correction bit for each coefficient in cm (zigzag positions), in order: the ones read as 1 go to corr
__device__ __forceinline__ int corrections(const uint8_t* __restrict__ buf, int pos, int end_bits, uint64_t cm,
                                           uint64_t& corr) {
  while (cm) {
    const int z = __ffsll((long long)cm) - 1;
    cm &= cm - 1;
    if (getbit(buf, pos++, end_bits)) corr |= 1ull << z;
  }
  return pos;
}

// One restart interval of an AC refinement scan: its n blocks from scan-order block q0, bits [pos, end_bits), up to
// scan-order block `limit`.  A block's non-zero history is a 64-bit zigzag mask taken at its start (coefficients made
// non-zero in this scan are never passed again in that block), a run is one __fns over the zero-history mask, and a
// block's changes are committed only once it decoded whole, and only if `write`.  Returns the failing block (invalid
// code, a size other than 0 or 1, a run past Se) relative to q0, or -1.
__device__ int refine_interval(const uint8_t* __restrict__ buf, int pos, int end_bits, const int* act, const PScan& p,
                               const Geom& g, int16_t* coef, int q0, int n, int limit, bool write) {
  const int p1 = 1 << p.al, m1 = -p1;
  const uint64_t band = (p.se == 63 ? ~0ull : (1ull << (p.se + 1)) - 1) & ~((1ull << p.ss) - 1);
  int eob = 0;
  for (int i = 0; i < n && q0 + i < limit; ++i) {
    if (eob == 0 && pos >= end_bits) break;
    int16_t* bc = coef + (size_t)scan_block(g, p, q0 + i) * 64;
    uint64_t nz = 0, corr = 0, add = 0, neg = 0;
    for (int z = p.ss; z <= p.se; ++z) nz |= (uint64_t)(bc[c_zigzag[z]] != 0) << z;
    int k = p.ss;
    if (eob == 0) {
      while (k <= p.se) {
        int l;
        const int sym = decode_sym(act, peek16(buf, pos, end_bits), l);
        if (sym < 0) return i;
        pos += l;
        const int r = sym >> 4, s = sym & 15;
        bool negative = false;
        if (s) {
          if (s != 1) return i;
          negative = !getbit(buf, pos++, end_bits);
        } else if (r != 15) {
          eob = (1 << r) + (r ? (int)(peek16(buf, pos, end_bits) >> (16 - r)) : 0);
          pos += r;
          break;
        }
        const uint64_t from_k = ~0ull << k;
        const uint64_t zeros = ~nz & band & from_k;
        if (__popcll(zeros) <= r) return i;
        const int t = nth_bit(zeros, r);
        pos = corrections(buf, pos, end_bits, nz & from_k & ((1ull << t) - 1), corr);
        if (s) {
          add |= 1ull << t;
          if (negative) neg |= 1ull << t;
        }
        k = t + 1;
      }
    }
    if (eob > 0) {
      if (k <= 63) pos = corrections(buf, pos, end_bits, nz & band & (~0ull << k), corr);
      --eob;
    }
    if (!write) continue;
    while (corr) {
      const int z = __ffsll((long long)corr) - 1;
      corr &= corr - 1;
      int16_t& c = bc[c_zigzag[z]];
      if ((c & p1) == 0) c = (int16_t)(c + (c >= 0 ? p1 : m1));
    }
    while (add) {
      const int z = __ffsll((long long)add) - 1;
      add &= add - 1;
      bc[c_zigzag[z]] = (int16_t)((neg >> z & 1) ? m1 : p1);
    }
  }
  return -1;
}

struct SegSat {   // segmented sum saturating at 2^30 (block counts of garbage paths can be large)
  __device__ __forceinline__ SegPair operator()(const SegPair& a, const SegPair& b) const {
    return SegPair{a.f | b.f, b.f ? b.v : min(a.v + b.v, 1u << 30)};
  }
};

__device__ __noinline__ void progressive_decode(const uint8_t* __restrict__ file, const int32_t* __restrict__ blk,
                                                const Geom& g, const JpegWs& L, uint8_t* base, int* tabs,
                                                typename ScanI::TempStorage& tmpi, typename ScanP::TempStorage& tmpp,
                                                int* sh_int) {
  const int tid = threadIdx.x;
  int32_t* stats = reinterpret_cast<int32_t*>(base + L.stats);
  int16_t* coef = reinterpret_cast<int16_t*>(base + L.coef);
  uint8_t* comp = base + L.comp;
  int32_t* seg_start = reinterpret_cast<int32_t*>(base + L.seg_start);
  int32_t* seg_total = reinterpret_cast<int32_t*>(base + L.seg_total);
  int32_t* sub_base = reinterpret_cast<int32_t*>(base + L.sub_base);
  int32_t* sub = reinterpret_cast<int32_t*>(base + L.sub);
  auto F = [&](int field, int t) -> int32_t& { return sub[(size_t)field * L.subs_cap + t]; };
  const int nsc = min(max(blk[10], 0), DEFER_JPEG_MAX_SCANS), ntab = min(max(blk[11], 0), DEFER_JPEG_MAX_TABLES);
  const int32_t* pool = blk + DEFER_JPEG_POOL_OFF;
  for (int i = tid; i < g.blocks * 8; i += JT) reinterpret_cast<uint4*>(coef)[i] = make_uint4(0, 0, 0, 0);
  int T = 0, R = 0, NS = 0, rounds = 0, done = 0, cutoff = g.blocks;
  for (int si = 0; si < nsc; ++si) {
    const PScan p = pscan(blk + DEFER_JPEG_SCAN_OFF + si * DEFER_JPEG_SCAN_INTS, g, ntab, L.slot);
    const bool dc = p.ss == 0, first = p.ah == 0;
    __syncthreads();                     // the previous scan is done with the tables, comp and the interval arrays
    if (!(dc && !first) && ntab == 0) {  // no table to read: the block declares none
      cutoff = 0;
      break;
    }
    for (int i = tid; i < HUFF; i += JT) {
      if (dc && first)
        for (int c = 0; c < (p.per > 1 ? 3 : 1); ++c) tabs[c * HUFF + i] = pool[(size_t)p.dct[c] * HUFF + i];
      if (!dc) tabs[3 * HUFF + i] = pool[(size_t)p.act * HUFF + i];
    }
    if (tid == 0) sh_int[1] = p.nq;      // the first scan-order block whose decode failed
    int t_n, r_n, nsubs;
    unstuff_intervals(file + p.off, p.len, p.nseg, comp, seg_start, seg_total, sub_base, L.subs_cap, tmpi, t_n, r_n,
                      nsubs);
    T += t_n;
    R += r_n;
    auto interval_of = [&](int q) { return p.ri ? q / p.per / p.ri : 0; };
    auto exp_of = [&](int k) { return (p.ri ? min(p.ri, p.units - k * p.ri) : p.units) * p.per; };
    if (dc && !first) {                  // DC refinement: bit i of an interval ORs 1 << Al into its block i
      for (int q = tid; q < p.nq; q += JT) {
        const int k = interval_of(q);
        const int bit = seg_start[k] * 8 + q - (p.ri ? k * p.ri * p.per : 0);
        if (getbit(comp, bit, seg_start[k + 1] * 8)) {
          int16_t* c0 = coef + (size_t)scan_block(g, p, q) * 64;
          *c0 = (int16_t)(*c0 | (1 << p.al));
        }
      }
    } else if (!first) {                 // AC refinement: one thread per interval; with several, a dry run finds the cut
      int limit = p.nq;
      for (int pass = p.nseg > 1 ? 0 : 1; pass < 2; ++pass) {
        for (int k = tid; k < p.nseg; k += JT) {
          const int q0 = p.ri ? k * p.ri : 0;
          const int f = refine_interval(comp, seg_start[k] * 8, seg_start[k + 1] * 8, tabs + 3 * HUFF, p, g, coef, q0,
                                        exp_of(k), limit, pass == 1);
          if (f >= 0) atomicMin(&sh_int[1], q0 + f);
        }
        __syncthreads();
        limit = sh_int[1];
      }
    } else {                             // DC first / AC first: self-synchronisation, as the baseline decode
      for (int t = tid; t < nsubs; t += JT) {
        int lo = 0, hi = p.nseg - 1;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (sub_base[mid] <= t) lo = mid; else hi = mid - 1;
        }
        const int a = seg_start[lo] * 8, e = seg_start[lo + 1] * 8;
        int pos = a + (t - sub_base[lo]) * S_BITS, jk = p.ss;
        const int end = min(pos + S_BITS, e);
        F(SUB_SEG, t) = lo;
        F(SUB_EPOS, t) = pos;
        F(SUB_EJK, t) = jk;
        F(SUB_CNT, t) = psync_run(comp, e, end, tabs, p, g, pos, jk);
        F(SUB_XPOS, t) = pos;
        F(SUB_XJK, t) = jk;
      }
      auto sub_end = [&](int t, int& seg_end) {
        const int k = F(SUB_SEG, t);
        seg_end = seg_start[k + 1] * 8;
        return min(seg_start[k] * 8 + (t - sub_base[k] + 1) * S_BITS, seg_end);
      };
      for (++rounds;; ++rounds) {
        __syncthreads();
        if (tid == 0) sh_int[0] = 0;
        for (int t = tid; t < nsubs; t += JT) {
          F(SUB_PPOS, t) = INT_MIN;
          if (t == 0 || F(SUB_SEG, t - 1) != F(SUB_SEG, t)) continue;
          const int np = F(SUB_XPOS, t - 1), njk = F(SUB_XJK, t - 1);
          if (np != F(SUB_EPOS, t) || njk != F(SUB_EJK, t)) {
            F(SUB_PPOS, t) = np;
            F(SUB_PJK, t) = njk;
          }
        }
        __syncthreads();
        for (int t = tid; t < nsubs; t += JT) {
          int pos = F(SUB_PPOS, t);
          if (pos == INT_MIN) continue;
          int jk = F(SUB_PJK, t);
          F(SUB_EPOS, t) = pos;
          F(SUB_EJK, t) = jk;
          int seg_end;
          const int end = sub_end(t, seg_end);
          F(SUB_CNT, t) = psync_run(comp, seg_end, end, tabs, p, g, pos, jk);
          F(SUB_XPOS, t) = pos;
          F(SUB_XJK, t) = jk;
          sh_int[0] = 1;
        }
        __syncthreads();
        if (!sh_int[0]) break;
      }
      NS += nsubs;
      // blocks before each subsequence within its interval: a segmented prefix sum
      unsigned carry = 0;
      for (int t0 = 0; t0 < nsubs; t0 += JT) {
        const int t = t0 + tid;
        SegPair in{t < nsubs && (t == 0 || F(SUB_SEG, t - 1) != F(SUB_SEG, t)), t < nsubs ? (unsigned)F(SUB_CNT, t) : 0u};
        SegPair out;
        ScanP(tmpp).InclusiveScan(in, out, SegSat());
        const unsigned sum = out.f ? out.v : min(carry + out.v, 1u << 30);
        if (t < nsubs) {
          F(SUB_PRE, t) = (int)(sum - in.v);
          if (t + 1 == nsubs || F(SUB_SEG, t + 1) != F(SUB_SEG, t))
            seg_total[F(SUB_SEG, t)] = (int)min(sum, (unsigned)exp_of(F(SUB_SEG, t)));
        }
        if (tid == JT - 1) sh_int[2] = (int)sum;
        __syncthreads();
        carry = (unsigned)sh_int[2];
        __syncthreads();
      }
      // write: each block by the subsequence it starts in; a DC first scan writes its differences
      for (int t = tid; t < nsubs; t += JT) {
        int pos = F(SUB_EPOS, t), seg_end;
        const int k_seg = F(SUB_SEG, t), end = sub_end(t, seg_end);
        int j = F(SUB_EJK, t) >> 8, k = F(SUB_EJK, t) & 255, z, v, eob;
        int idx = F(SUB_PRE, t);
        bool ok = true;
        while (k != p.ss) {              // the tail of a block that started in the predecessor
          if (!pstep(comp, seg_end, tabs, p, g, j, pos, k, z, v, eob)) { ok = false; break; }
          idx += eob;
          if (k > p.se) k = p.ss, j = j + 1 == p.per ? 0 : j + 1;
        }
        if (!ok) continue;
        const int exp_k = exp_of(k_seg), q0 = p.ri ? k_seg * p.ri * p.per : 0;
        while (pos < end && idx < exp_k) {
          const int q = q0 + idx;
          int16_t* out = coef + (size_t)scan_block(g, p, q) * 64;
          int extra = 0;
          do {
            if (!pstep(comp, seg_end, tabs, p, g, j, pos, k, z, v, eob)) { ok = false; break; }
            extra += eob;
            if (z == 0 && dc) out[0] = (int16_t)v;
            else if (z >= 0) out[c_zigzag[z]] = (int16_t)((unsigned)v << p.al);
          } while (k <= p.se);
          if (!ok) {
            atomicMin(&sh_int[1], q);
            break;
          }
          k = p.ss;
          j = j + 1 == p.per ? 0 : j + 1;
          idx += 1 + extra;
        }
      }
      __syncthreads();
      const int cut = sh_int[1];
      if (dc) {                          // DC prediction per component, in scan order, restarting with each interval
        for (int c = p.per > 1 ? 0 : p.comp; c < (p.per > 1 ? g.ncomp : p.comp + 1); ++c) {
          const int nbc = p.per > 1 && c == 0 ? g.nb0 : 1, offc = p.per > 1 && c > 0 ? g.nb0 + c - 1 : 0;
          const int nq = p.units * nbc;
          unsigned carry2 = 0;
          for (int q0 = 0; q0 < nq; q0 += JT) {
            const int q = q0 + tid;
            int b = 0;
            bool valid = false;
            SegPair in{0, 0u};
            if (q < nq) {
              const int u = q / nbc, ks = p.ri ? u / p.ri : 0;
              const int sq = u * p.per + offc + q % nbc;
              b = scan_block(g, p, sq);
              in.f = q % nbc == 0 && (p.ri ? u % p.ri == 0 : u == 0);
              valid = sq < cut && sq - (p.ri ? ks * p.ri * p.per : 0) < seg_total[ks];
              in.v = valid ? (unsigned)(int)coef[(size_t)b * 64] : 0u;
            }
            SegPair out;
            __syncthreads();
            ScanP(tmpp).InclusiveScan(in, out, SegSum());
            const unsigned sum = out.f ? out.v : carry2 + out.v;
            __syncthreads();
            if (q < nq) coef[(size_t)b * 64] = valid ? (int16_t)(int)(sum << p.al) : (int16_t)0;
            if (tid == JT - 1) sh_int[2] = (int)sum;
            __syncthreads();
            carry2 = (unsigned)sh_int[2];
          }
        }
      } else if (cut < p.nq) {           // an AC first scan gives nothing from the failing block on
        for (int q = cut + tid; q < p.nq; q += JT) {
          int16_t* out = coef + (size_t)scan_block(g, p, q) * 64;
          for (int z = p.ss; z <= p.se; ++z) out[c_zigzag[z]] = 0;
        }
      }
    }
    __syncthreads();
    const int cut = sh_int[1];
    if (cut < p.nq) {
      cutoff = cut;
      break;
    }
    ++done;
  }
  if (tid == 0) {
    stats[0] = T;
    stats[1] = R;
    stats[2] = NS;
    stats[3] = rounds;
    stats[4] = cutoff;
    stats[5] = done;
  }
}

__global__ void __launch_bounds__(JT) jpeg_entropy_kernel(const uint8_t* __restrict__ files, const int32_t* __restrict__ blocks,
                                                          uint8_t* __restrict__ ws, int H, int W, JpegWs L) {
  __shared__ union {
    typename ScanI::TempStorage i;
    typename ScanP::TempStorage p;
  } tmp;
  __shared__ int tabs[6 * HUFF];
  __shared__ int sh_int[8];
  const int s = blockIdx.x, tid = threadIdx.x;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const Geom g = geom(blk, H, W, L.slot);
  uint8_t* base = ws + (size_t)s * L.stride;
  int32_t* stats = reinterpret_cast<int32_t*>(base + L.stats);
  int16_t* coef = reinterpret_cast<int16_t*>(base + L.coef);
  uint8_t* comp = base + L.comp;
  int32_t* seg_start = reinterpret_cast<int32_t*>(base + L.seg_start);
  int32_t* seg_total = reinterpret_cast<int32_t*>(base + L.seg_total);
  int32_t* sub_base = reinterpret_cast<int32_t*>(base + L.sub_base);
  int32_t* sub = reinterpret_cast<int32_t*>(base + L.sub);
  auto F = [&](int field, int t) -> int32_t& { return sub[(size_t)field * L.subs_cap + t]; };
  if (blk[10] != 0) {
    progressive_decode(files + (size_t)s * L.file, blk, g, L, base, tabs, tmp.i, tmp.p, sh_int);
    return;
  }
  for (int i = tid; i < 6 * HUFF; i += JT) tabs[i] = blk[T_OFF + i];
  int T, R, nsubs;
  unstuff_intervals(files + (size_t)s * L.file + g.off, g.len, g.nseg, comp, seg_start, seg_total, sub_base, L.subs_cap,
                    tmp.i, T, R, nsubs);
  // ---- 3. every subsequence decodes from the default state at its first bit
  for (int t = tid; t < nsubs; t += JT) {
    int lo = 0, hi = g.nseg - 1;          // the last interval whose first subsequence is <= t
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (sub_base[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const int a = seg_start[lo] * 8, e = seg_start[lo + 1] * 8;
    int pos = a + (t - sub_base[lo]) * S_BITS, jk = 0;
    const int end = min(pos + S_BITS, e);
    F(SUB_SEG, t) = lo;
    F(SUB_EPOS, t) = pos;
    F(SUB_EJK, t) = 0;
    F(SUB_CNT, t) = sync_run(comp, e, end, tabs, g, pos, jk);
    F(SUB_XPOS, t) = pos;
    F(SUB_XJK, t) = jk;
  }
  // ---- 4. synchronise: a subsequence whose predecessor (same interval) left in another state than it entered re-decodes
  //         from there; until no entry changes.  The first subsequence of an interval starts at a known state.
  int rounds = 1;
  auto sub_end = [&](int t, int& seg_end) {
    const int k = F(SUB_SEG, t);
    seg_end = seg_start[k + 1] * 8;
    return min(seg_start[k] * 8 + (t - sub_base[k] + 1) * S_BITS, seg_end);
  };
  for (;;) {
    __syncthreads();
    if (tid == 0) sh_int[0] = 0;
    for (int t = tid; t < nsubs; t += JT) {
      F(SUB_PPOS, t) = INT_MIN;
      if (t == 0 || F(SUB_SEG, t - 1) != F(SUB_SEG, t)) continue;
      const int np = F(SUB_XPOS, t - 1), njk = F(SUB_XJK, t - 1);
      if (np != F(SUB_EPOS, t) || njk != F(SUB_EJK, t)) {
        F(SUB_PPOS, t) = np;
        F(SUB_PJK, t) = njk;
      }
    }
    __syncthreads();
    for (int t = tid; t < nsubs; t += JT) {
      int pos = F(SUB_PPOS, t);
      if (pos == INT_MIN) continue;
      int jk = F(SUB_PJK, t);
      F(SUB_EPOS, t) = pos;
      F(SUB_EJK, t) = jk;
      int seg_end;
      const int end = sub_end(t, seg_end);
      F(SUB_CNT, t) = sync_run(comp, seg_end, end, tabs, g, pos, jk);
      F(SUB_XPOS, t) = pos;
      F(SUB_XJK, t) = jk;
      sh_int[0] = 1;
    }
    __syncthreads();
    if (!sh_int[0]) break;
    ++rounds;
  }
  // ---- 5. block positions: prefix sum of the blocks each subsequence starts
  {
    int carry = 0;
    for (int t0 = 0; t0 < nsubs; t0 += JT) {
      const int t = t0 + tid;
      int pre, tot;
      ScanI(tmp.i).ExclusiveSum(t < nsubs ? F(SUB_CNT, t) : 0, pre, tot);
      if (t < nsubs) F(SUB_PRE, t) = carry + pre;
      carry += tot;
      __syncthreads();
    }
  }
  if (tid == 0) sh_int[1] = g.blocks;    // first block that did not decode (cutoff)
  __syncthreads();
  for (int t = tid; t < nsubs; t += JT) {
    const int k = F(SUB_SEG, t);
    const int exp_k = (g.ri ? min(g.ri, g.mcus - k * g.ri) : g.mcus) * g.bpm;
    const int done = F(SUB_PRE, t) - F(SUB_PRE, sub_base[k]);
    if (t + 1 == nsubs || F(SUB_SEG, t + 1) != k) seg_total[k] = min(done + F(SUB_CNT, t), exp_k);
  }
  // ---- 6. write the coefficients: each block by the subsequence it starts in, all 64 values, zero runs included
  for (int t = tid; t < nsubs; t += JT) {
    int pos = F(SUB_EPOS, t);
    const int k_seg = F(SUB_SEG, t);
    int seg_end;
    const int end = sub_end(t, seg_end);
    int j = F(SUB_EJK, t) >> 8, k = F(SUB_EJK, t) & 255, z, v;
    bool ok = true;
    while (k != 0) {                     // the tail of a block that started in the predecessor
      const int c = comp_of(g, j);
      if (!jstep(comp, seg_end, tabs + c * HUFF, tabs + (3 + c) * HUFF, pos, k, z, v)) { ok = false; break; }
      if (k >= 64) k = 0, j = j + 1 == g.bpm ? 0 : j + 1;
    }
    if (!ok) continue;
    const int exp_k = (g.ri ? min(g.ri, g.mcus - k_seg * g.ri) : g.mcus) * g.bpm;
    const int first = g.ri ? k_seg * g.ri * g.bpm : 0;
    int idx = F(SUB_PRE, t) - F(SUB_PRE, sub_base[k_seg]);
    while (pos < end && idx < exp_k) {
      const int b = first + idx;
      int16_t* out = coef + (size_t)b * 64;
      const int c = comp_of(g, j);
      do {
        const int k0 = k;
        if (!jstep(comp, seg_end, tabs + c * HUFF, tabs + (3 + c) * HUFF, pos, k, z, v)) { ok = false; break; }
        for (int q = k0; q < k; ++q) out[c_zigzag[q]] = (int16_t)(q == z ? v : 0);
      } while (k < 64);
      if (!ok) {
        atomicMin(&sh_int[1], b);
        break;
      }
      k = 0;
      j = j + 1 == g.bpm ? 0 : j + 1;
      ++idx;
    }
  }
  __syncthreads();
  const int cutoff = sh_int[1];
  // ---- 7. DC prediction: per component, a prefix sum in int32 segmented by restart interval; blocks that did not decode
  //         are zero
  for (int c = 0; c < g.ncomp; ++c) {
    const int nbc = c == 0 ? g.nb0 : 1, offc = c == 0 ? 0 : g.nb0 + c - 1;
    const int nq = g.mcus * nbc;
    unsigned carry = 0;
    for (int q0 = 0; q0 < nq; q0 += JT) {
      const int q = q0 + tid;
      int b = 0;
      bool valid = false;
      SegPair in{0, 0u};
      if (q < nq) {
        const int m = q / nbc, kseg = g.ri ? m / g.ri : 0;
        b = m * g.bpm + offc + q % nbc;
        in.f = q % nbc == 0 && (g.ri ? m % g.ri == 0 : m == 0);
        valid = b < cutoff && b - (g.ri ? kseg * g.ri * g.bpm : 0) < seg_total[kseg];
        in.v = valid ? (unsigned)(int)coef[(size_t)b * 64] : 0u;
      }
      SegPair out;
      __syncthreads();
      ScanP(tmp.p).InclusiveScan(in, out, SegSum());
      const unsigned sum = out.f ? out.v : carry + out.v;
      __syncthreads();
      if (q < nq) {
        int16_t* blkc = coef + (size_t)b * 64;
        if (valid) {
          blkc[0] = (int16_t)(int)sum;
        } else {
          for (int i = 0; i < 64; ++i) blkc[i] = 0;
        }
      }
      if (tid == JT - 1) sh_int[2] = (int)sum;
      __syncthreads();
      carry = (unsigned)sh_int[2];
    }
  }
  if (tid == 0) {
    stats[0] = T;
    stats[1] = R;
    stats[2] = nsubs;
    stats[3] = rounds;
    stats[4] = cutoff;
  }
}

// jidctint.c's ISLOW butterflies on one column (pass 1, descale by CONST_BITS - PASS1_BITS, stored as int) or one row
// (pass 2, descale by CONST_BITS + PASS1_BITS + 3)
__device__ __forceinline__ void idct_1d(const long long* s, long long* o, int sh) {
  long long z2 = s[2], z3 = s[6];
  long long z1 = (z2 + z3) * 4433;
  const long long tmp2e = z1 + z3 * -15137, tmp3e = z1 + z2 * 6270;
  const long long t0 = (s[0] + s[4]) * 8192, t1 = (s[0] - s[4]) * 8192;
  const long long t10 = t0 + tmp3e, t13 = t0 - tmp3e, t11 = t1 + tmp2e, t12 = t1 - tmp2e;
  long long tmp0 = s[7], tmp1 = s[5], tmp2 = s[3], tmp3 = s[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * 9633;
  tmp0 *= 2446;
  tmp1 *= 16819;
  tmp2 *= 25172;
  tmp3 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  const long long r = 1ll << (sh - 1);
  o[0] = (t10 + tmp3 + r) >> sh;
  o[7] = (t10 - tmp3 + r) >> sh;
  o[1] = (t11 + tmp2 + r) >> sh;
  o[6] = (t11 - tmp2 + r) >> sh;
  o[2] = (t12 + tmp1 + r) >> sh;
  o[5] = (t12 - tmp1 + r) >> sh;
  o[3] = (t13 + tmp0 + r) >> sh;
  o[4] = (t13 - tmp0 + r) >> sh;
}

constexpr int IDCT_BLOCKS = 16;   // 8x8 blocks per CTA, 8 threads each

__global__ void __launch_bounds__(IDCT_BLOCKS * 8) jpeg_idct_kernel(const int32_t* __restrict__ blocks, uint8_t* __restrict__ ws,
                                                                    int H, int W, JpegWs L) {
  __shared__ int wsp[IDCT_BLOCKS][64];
  const int s = blockIdx.y, lb = threadIdx.x >> 3, r = threadIdx.x & 7;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const Geom g = geom(blk, H, W, L.slot);
  const int b = blockIdx.x * IDCT_BLOCKS + lb;
  if (b >= g.blocks) return;               // the 8 threads of a block leave together
  const unsigned grp = 0xFFu << (threadIdx.x & 24);
  uint8_t* base = ws + (size_t)s * L.stride;
  const int16_t* cf = reinterpret_cast<const int16_t*>(base + L.coef) + (size_t)b * 64;
  const int m = b / g.bpm, j = b % g.bpm, c = comp_of(g, j);
  const int mx = m % g.mcux, my = m / g.mcux;
  const int bx = c == 0 ? mx * g.hs + j % g.hs : mx, by = c == 0 ? my * g.vs + j / g.hs : my;
  const int32_t* q = blk + Q_OFF + 64 * c;
  long long in[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) in[k] = (long long)cf[k * 8 + r] * (long long)q[k * 8 + r];
  idct_1d(in, o, 11);
#pragma unroll
  for (int k = 0; k < 8; ++k) wsp[lb][k * 8 + r] = (int)o[k];
  __syncwarp(grp);
#pragma unroll
  for (int k = 0; k < 8; ++k) in[k] = wsp[lb][r * 8 + k];
  idct_1d(in, o, 18);
  uint32_t px[2] = {0, 0};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int v = (int)(((o[k] & 1023) ^ 512) - 512) + 128;   // idct_range_limit[x & RANGE_MASK]
    px[k >> 2] |= (uint32_t)min(max(v, 0), 255) << (8 * (k & 3));
  }
  const int rs = g.bw[c] * 8;
  uint8_t* dst = base + L.planes + g.poff[c] + (size_t)(by * 8 + r) * rs + bx * 8;
  *reinterpret_cast<uint2*>(dst) = make_uint2(px[0], px[1]);
}

// chroma sample at output pixel (x, y) of a plane downsampled by (hs, vs): libjpeg-turbo's h2v1 / h2v2 fancy upsampling
// when the downsampled width exceeds 2, else replication
__device__ __forceinline__ int upsample(const uint8_t* __restrict__ p, int rs, int x, int y, int h, int w, int hs, int vs) {
  if (hs == 1) return p[(size_t)y * rs + x];
  const int dw = (w + 1) >> 1, i = x >> 1, odd = x & 1;
  if (dw <= 2) return p[(size_t)(y / vs) * rs + i];
  const int in_ = odd ? min(i + 1, dw - 1) : max(i - 1, 0);
  if (vs == 1) {
    const uint8_t* row = p + (size_t)y * rs;
    const int a = row[i], n = row[in_];
    if (odd) return i == dw - 1 ? a : (3 * a + n + 2) >> 2;
    return i == 0 ? a : (3 * a + n + 1) >> 2;
  }
  const int dh = (h + 1) >> 1, r0 = y >> 1, r1 = (y & 1) ? min(r0 + 1, dh - 1) : max(r0 - 1, 0);
  const uint8_t* p0 = p + (size_t)r0 * rs;
  const uint8_t* p1 = p + (size_t)r1 * rs;
  const int cs = 3 * p0[i] + p1[i], cn = 3 * p0[in_] + p1[in_];
  if (odd) return i == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + cn + 7) >> 4;
  return i == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + cn + 8) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const int32_t* __restrict__ blocks, const uint8_t* __restrict__ ws,
                                                         uint8_t* __restrict__ y_out, int H, int W, JpegWs L) {
  const int s = blockIdx.y;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const Geom g = geom(blk, H, W, L.slot);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.h * g.w) return;
  const int x = i % g.w, y = i / g.w;
  const uint8_t* pl = ws + (size_t)s * L.stride + L.planes;
  const int Y = pl[g.poff[0] + (size_t)y * g.bw[0] * 8 + x];
  uint8_t* o = y_out + (size_t)s * L.slot + (size_t)i * 3;
  if (g.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int rs = g.bw[1] * 8;
  const int cb = upsample(pl + g.poff[1], rs, x, y, g.h, g.w, g.hs, g.vs) - 128;
  const int cr = upsample(pl + g.poff[2], rs, x, y, g.h, g.w, g.hs, g.vs) - 128;
  // jdcolor.c: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554, SCALEBITS 16
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  o[0] = (uint8_t)min(max(R, 0), 255);
  o[1] = (uint8_t)min(max(G, 0), 255);
  o[2] = (uint8_t)min(max(B, 0), 255);
}

}  // namespace

size_t jpeg_workspace_bytes(int H, int W, int n) { return jpeg_ws(H, W).stride * (size_t)n; }

size_t jpeg_ws_stride(int H, int W, size_t* coef_off, size_t* plane_off) {
  const JpegWs L = jpeg_ws(H, W);
  if (coef_off) *coef_off = L.coef;
  if (plane_off) *plane_off = L.planes;
  return L.stride;
}

// Bit positions in the entropy kernel are ints: the last subsequence's end, up to slot * 8 + S_BITS, must fit in one
bool jpeg_bound_ok(int H, int W) { return (uint64_t)H * W * 3 * 8 + S_BITS < (1ull << 31); }

int launch_jpeg_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                       cudaStream_t st, const DecodeStrides* strides) {
  JpegWs L = jpeg_ws(H, W);
  if (strides) {
    L.file = strides->file;
    L.stride = strides->ws;
    L.block_ints = strides->block_ints;
    L.take = strides->take;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  prefer_max_smem(jpeg_entropy_kernel);
  jpeg_entropy_kernel<<<n, JT, 0, st>>>(files, blocks, ws, H, W, L);
  prefer_max_smem(jpeg_idct_kernel);
  jpeg_idct_kernel<<<dim3((unsigned)((L.blocks_cap + IDCT_BLOCKS - 1) / IDCT_BLOCKS), (unsigned)n), IDCT_BLOCKS * 8, 0, st>>>(
      blocks, ws, H, W, L);
  prefer_max_smem(jpeg_color_kernel);
  jpeg_color_kernel<<<dim3((unsigned)(((size_t)H * W + 255) / 256), (unsigned)n), 256, 0, st>>>(blocks, ws, y, H, W, L);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

}  // namespace defer

using namespace defer;

extern "C" {

int defer_k_jpeg_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* coef_off,
                           uint64_t* plane_off) {
  DEFER_CHECK(H >= 1 && W >= 1 && n >= 1 && jpeg_bound_ok(H, W),
              "k_jpeg_workspace: bad bound %dx%d (n %d)", H, W, n);
  const JpegWs L = jpeg_ws(H, W);
  if (bytes) *bytes = L.stride * (uint64_t)n;
  if (sample_stride) *sample_stride = L.stride;
  if (coef_off) *coef_off = L.coef;
  if (plane_off) *plane_off = L.planes;
  return DEFER_OK;
}

int defer_k_jpeg_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                        void* stream) {
  DEFER_CHECK(files && blocks && workspace && y, "k_jpeg_decode: null pointer");
  DEFER_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1 && jpeg_bound_ok(H, W),
              "k_jpeg_decode: bad sizes (n %d, bound %dx%d)", n, H, W);
  DEFER_CHECK(((uintptr_t)blocks & 3) == 0 && ((uintptr_t)workspace & 255) == 0,
              "k_jpeg_decode: blocks must be 4-byte and the workspace 256-byte aligned");
  return launch_jpeg_decode(files, blocks, n, H, W, workspace, y, (cudaStream_t)stream);
}

}  // extern "C"
