// png.cu - DEFER_OP_PNG_DECODE: non-interlaced PNG files decoded on the GPU, bit for bit as Pillow's convert("RGB") gives
// them, and as defer_b200/png.py restates it (with its one defined result for corrupt data).  Three kernels per
// microbatch, each with a fixed grid sized from the slot bound (H, W) and an early exit per sample:
//   png_inflate_kernel   one CTA per sample: all its threads gather the IDAT payloads into one zlib stream, then warp 0
//                        inflates it into the raw scanlines.  The symbol decode is serial: every lane of the warp runs
//                        the same decoder on the same bits (uniform loads, no shuffles), lane 0 stores literals, and
//                        the whole warp copies stored blocks and matches.  Huffman tables are built by the warp in
//                        shared memory: a 10-bit lookahead table, then a canonical count / symbol walk (puff.c's) for
//                        longer codes.
//   png_unfilter_kernel  one CTA per sample, one thread per row in bands of UT rows: a wavefront in which row r works
//                        on pixel x while row r - 1 works on x + 1, as Paeth reads the left, up and up-left neighbours
//   png_expand_kernel    Pillow's conversion of the file's mode and depth to RGB, one thread per pixel, packed
//                        (h, w, 3) at the start of the sample's U8 slot
// Nothing here trusts the per-sample block: size, colour type and depth are clamped to valid ones, IDAT ranges into
// the slot and the gathered stream into its workspace, so a stale, zero or corrupt block gives wrong pixels, never an
// access outside the sample's slot, workspace or image.  Every loop is bounded: the inflate consumes at least one bit of
// the gathered stream per pass or ends, and a match or stored block never writes past h * (1 + bytes per row).
#include "common.cuh"

namespace defer {

// Per-sample workspace layout (byte offsets from the sample's base); host and device compute it the same way.
struct PngWs {
  size_t slot, stats, stream, raw, stride;   // slot: the extent clamp of a file
  size_t file;                               // the file slot stride (DecodeStrides)
  int block_ints;                            // the block stride
  int take;                                  // which samples (decode_takes)
};

__host__ __device__ inline PngWs png_ws(int H, int W) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  PngWs L;
  L.slot = DEFER_PNG_SLOT_BYTES((size_t)H, (size_t)W);
  size_t o = 0;
  L.stats = o;   o += 256;                                  // int32 status, bytes produced, rows of unknown filter type
  L.stream = o;  o += al(L.slot + 64);                      // the gathered zlib stream, zero past its end
  L.raw = o;     o += al((size_t)H * (1 + 8 * (size_t)W));  // the scanlines, unfiltered in place
  L.stride = o;
  L.file = L.slot;
  L.block_ints = DEFER_PNG_BLOCK_INTS;
  L.take = 0;
  return L;
}

namespace {

constexpr int IT = 128;          // threads of the inflate kernel (gather); warp 0 inflates
constexpr int UT = 256;          // threads (rows per band) of the unfilter kernel
constexpr int LUT_BITS = 10;     // lookahead bits of the literal/length and distance tables
constexpr unsigned FULL = 0xffffffffu;

enum { ST_OK = 0, ST_SHORT = 1, ST_EXHAUSTED = 2, ST_BAD_BLOCK = 3, ST_BAD_HEADER = 4, ST_BAD_SYMBOL = 5,
       ST_BAD_DISTANCE = 6, ST_RUNNING = -1 };

__constant__ uint16_t c_lbase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                     31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                     193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Geometry of one sample from its block header, clamped into the slot (H, W) and to a valid colour type and depth.
struct PGeom {
  int h, w, ct, depth, ch, bpr, bpp, nidat;
  long long raw;   // h * (1 + bpr): the scanline bytes
};

__device__ __forceinline__ PGeom pgeom(const int32_t* blk, int H, int W) {
  PGeom g;
  g.h = min(max(blk[0], 1), H);
  g.w = min(max(blk[1], 1), W);
  const int ct = blk[2], d = blk[3];
  g.ct = (ct == 2 || ct == 3 || ct == 4 || ct == 6) ? ct : 0;
  g.ch = g.ct == 2 ? 3 : g.ct == 4 ? 2 : g.ct == 6 ? 4 : 1;
  const bool low = d == 1 || d == 2 || d == 4;
  g.depth = (d == 8 || (d == 16 && g.ct != 3) || (low && (g.ct == 0 || g.ct == 3))) ? d : 8;
  g.bpr = (int)(((long long)g.w * g.ch * g.depth + 7) / 8);
  g.bpp = max(1, g.ch * g.depth / 8);
  g.nidat = min(max(blk[6], 0), DEFER_PNG_MAX_IDAT);
  g.raw = (long long)g.h * (1 + g.bpr);
  return g;
}

// Huffman tables of the block being decoded (shared memory of warp 0).
struct Tables {
  uint16_t lut[2][1 << LUT_BITS];   // literal/length, distance: code length << 9 | symbol for codes of <= LUT_BITS bits
  uint16_t count[3][16];            // codes per length: literal/length, distance, code-length code
  uint16_t sym[2][288];             // symbols in canonical order
  uint16_t clsym[19];
  uint16_t offs[16], next[16];      // build scratch: first index and next code per length
  uint8_t lens[320];                // code lengths: literal/length then distance (or the 19 of the code-length code)
};

// 32 bits of the stream from bit `pos` (LSB first); the stream is 8-byte aligned and zero past its end
__device__ __forceinline__ uint32_t peek32(const uint8_t* st, long long pos) {
  const uint64_t* w = reinterpret_cast<const uint64_t*>(st);
  const long long q = pos >> 6;
  const int sh = (int)(pos & 63);
  const uint64_t lo = w[q], hi = w[q + 1];
  return (uint32_t)(sh ? (lo >> sh) | (hi << (64 - sh)) : lo);
}

// Build the canonical code of lens[0, n) into count / sym (and lut): true when zlib's inflate_table accepts it
// (not over-subscribed; incomplete only with a longest code of one bit, and never for the code-length code, which
// must have codes).  Every lane returns the same value.
__device__ bool build_code(Tables& t, const uint8_t* lens, int n, uint16_t* count, uint16_t* sym, uint16_t* lut, bool cl,
                           int lane) {
  if (lane < 16) count[lane] = 0;
  __syncwarp();
  for (int c = 0; c < n; c += 32) {
    const int i = c + lane;
    const int l = i < n ? lens[i] : 0;
    const unsigned m = __match_any_sync(FULL, l);
    if (l && lane == __ffs(m) - 1) count[l] += __popc(m);
    __syncwarp();
  }
  int left = 1, longest = 0;
  bool ok = true;
  for (int l = 1; l < 16; ++l) {
    left = 2 * left - count[l];
    if (left < 0) ok = false;
    if (count[l]) longest = l;
  }
  if (!ok || (cl && longest == 0) || (left > 0 && longest != 0 && (cl || longest != 1))) return false;
  if (lane == 0) {
    int o = 0, code = 0;
    for (int l = 1; l < 16; ++l) {
      code = (code + count[l - 1]) << 1;   // count[0] is 0
      t.offs[l] = (uint16_t)o;
      t.next[l] = (uint16_t)code;
      o += count[l];
    }
  }
  if (lut)
    for (int e = lane; e < (1 << LUT_BITS) / 2; e += 32) reinterpret_cast<uint32_t*>(lut)[e] = 0;
  __syncwarp();
  for (int c = 0; c < n; c += 32) {
    const int i = c + lane;
    const int l = i < n ? lens[i] : 0;
    const unsigned m = __match_any_sync(FULL, l);
    const int rank = __popc(m & ((1u << lane) - 1));
    if (l) {
      sym[t.offs[l] + rank] = (uint16_t)i;
      if (lut && l <= LUT_BITS) {
        const int rev = (int)(__brev((unsigned)(t.next[l] + rank)) >> (32 - l));
        for (int k = rev; k < (1 << LUT_BITS); k += 1 << l) lut[k] = (uint16_t)((l << 9) | i);
      }
    }
    __syncwarp();
    if (l && lane == __ffs(m) - 1) {
      t.offs[l] += __popc(m);
      t.next[l] += __popc(m);
    }
    __syncwarp();
  }
  return true;
}

// Decode one symbol at `pos`: the symbol, or -1 with `status` set (no code of the table, or its bits past the end)
__device__ __forceinline__ int decode_sym(const uint8_t* st, long long& pos, long long nbits, const uint16_t* lut,
                                          const uint16_t* count, const uint16_t* sym, int& status) {
  const uint32_t v = peek32(st, pos);
  if (lut) {
    const int e = lut[v & ((1u << LUT_BITS) - 1)];
    if (e) {
      const int l = e >> 9;
      if (pos + l > nbits) {
        status = ST_EXHAUSTED;
        return -1;
      }
      pos += l;
      return e & 511;
    }
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (v >> (l - 1)) & 1;
    const int c = count[l];
    if (code - first < c) {
      if (pos + l > nbits) {
        status = ST_EXHAUSTED;
        return -1;
      }
      pos += l;
      return sym[index + code - first];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  status = ST_BAD_SYMBOL;
  return -1;
}

// `n` bits at `pos` (n <= 16), or -1 with `status` = exhausted
__device__ __forceinline__ int take_bits(const uint8_t* st, long long& pos, long long nbits, int n, int& status) {
  if (pos + n > nbits) {
    status = ST_EXHAUSTED;
    return -1;
  }
  const int v = (int)(peek32(st, pos) & ((1u << n) - 1));
  pos += n;
  return v;
}

// A dynamic block's header: the code lengths, then both tables.  ST_RUNNING on success.
__device__ int read_dynamic(Tables& t, const uint8_t* st, long long& pos, long long nbits, int lane) {
  int status = ST_RUNNING;
  if (pos + 14 > nbits) return ST_EXHAUSTED;
  const uint32_t v = peek32(st, pos);
  pos += 14;
  const int hlit = (int)(v & 31) + 257, hdist = (int)((v >> 5) & 31) + 1, hclen = (int)((v >> 10) & 15) + 4;
  if (hlit > 286 || hdist > 30) return ST_BAD_HEADER;
  if (pos + 3 * hclen > nbits) return ST_EXHAUSTED;
  if (lane < 19) t.lens[c_clorder[lane]] = lane < hclen ? (uint8_t)((peek32(st, pos + 3 * lane)) & 7) : 0;
  pos += 3 * hclen;
  __syncwarp();
  if (!build_code(t, t.lens, 19, t.count[2], t.clsym, nullptr, true, lane)) return ST_BAD_HEADER;
  __syncwarp();
  const int total = hlit + hdist;
  int i = 0, prev = 0;
  while (i < total) {   // each pass consumes at least one bit or returns
    const int s = decode_sym(st, pos, nbits, nullptr, t.count[2], t.clsym, status);
    if (s < 0) return status;
    int val, rep;
    if (s < 16) {
      val = s;
      rep = 1;
    } else if (s == 16) {
      if (i == 0) return ST_BAD_HEADER;
      const int b = take_bits(st, pos, nbits, 2, status);
      if (b < 0) return status;
      val = prev;
      rep = 3 + b;
    } else {
      const int b = take_bits(st, pos, nbits, s == 17 ? 3 : 7, status);
      if (b < 0) return status;
      val = 0;
      rep = (s == 17 ? 3 : 11) + b;
    }
    if (i + rep > total) return ST_BAD_HEADER;
    __syncwarp();
    for (int k = lane; k < rep; k += 32) t.lens[i + k] = (uint8_t)val;
    i += rep;
    prev = val;
  }
  __syncwarp();
  if (t.lens[256] == 0) return ST_BAD_HEADER;
  if (!build_code(t, t.lens, hlit, t.count[0], t.sym[0], t.lut[0], false, lane)) return ST_BAD_HEADER;
  if (!build_code(t, t.lens + hlit, hdist, t.count[1], t.sym[1], t.lut[1], false, lane)) return ST_BAD_HEADER;
  __syncwarp();
  return ST_RUNNING;
}

__device__ void build_fixed(Tables& t, int lane) {
  for (int i = lane; i < 320; i += 32) t.lens[i] = (uint8_t)(i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5);
  __syncwarp();
  build_code(t, t.lens, 288, t.count[0], t.sym[0], t.lut[0], false, lane);
  build_code(t, t.lens + 288, 32, t.count[1], t.sym[1], t.lut[1], false, lane);
  __syncwarp();
}

// Inflate the gathered stream (all lanes of one warp run it in lockstep) into out[0, limit); returns (status, bytes)
__device__ int inflate_warp(Tables& t, const uint8_t* st, long long nbits, uint8_t* out, long long limit, long long& produced,
                            int lane) {
  long long pos = 16;   // past the zlib header (checked by the parser)
  int status = ST_RUNNING, tables = 0;   // tables: 1 = the fixed code is built
  produced = 0;
  while (status == ST_RUNNING) {
    if (pos + 3 > nbits) return ST_EXHAUSTED;
    const uint32_t hdr = peek32(st, pos) & 7;
    pos += 3;
    const int final = hdr & 1, type = hdr >> 1;
    if (type == 0) {
      pos = (pos + 7) & ~7ll;
      if (pos + 32 > nbits) return ST_EXHAUSTED;
      const uint32_t v = peek32(st, pos);
      pos += 32;
      const uint32_t len = v & 0xffff;
      if (len != (~(v >> 16) & 0xffff)) return ST_BAD_BLOCK;
      if (pos + 8ll * len > nbits) return ST_EXHAUSTED;
      const long long n = min((long long)len, limit - produced);
      const uint8_t* src = st + (pos >> 3);
      for (long long i = lane; i < n; i += 32) out[produced + i] = src[i];
      __syncwarp();
      produced += n;
      pos += 8ll * len;
      if (produced == limit) return ST_OK;
    } else if (type == 3) {
      return ST_BAD_BLOCK;
    } else {
      if (type == 1) {
        if (tables != 1) build_fixed(t, lane);
        tables = 1;
      } else {
        tables = 2;
        const int r = read_dynamic(t, st, pos, nbits, lane);
        if (r != ST_RUNNING) return r;
      }
      while (true) {   // each pass consumes at least one bit or returns
        int s = decode_sym(st, pos, nbits, t.lut[0], t.count[0], t.sym[0], status);
        if (s < 0) return status;
        if (s < 256) {
          if (lane == 0) out[produced] = (uint8_t)s;
          if (++produced == limit) return ST_OK;
          continue;
        }
        if (s == 256) break;
        s -= 257;
        if (s >= 29) return ST_BAD_SYMBOL;
        const int lb = take_bits(st, pos, nbits, c_lext[s], status);
        if (lb < 0) return status;
        const int length = c_lbase[s] + lb;
        const int ds = decode_sym(st, pos, nbits, t.lut[1], t.count[1], t.sym[1], status);
        if (ds < 0) return status;
        if (ds >= 30) return ST_BAD_SYMBOL;
        const int db = take_bits(st, pos, nbits, c_dext[ds], status);
        if (db < 0) return status;
        const int dist = c_dbase[ds] + db;
        if (dist > produced) return ST_BAD_DISTANCE;
        const int n = (int)min((long long)length, limit - produced);
        __syncwarp();   // lane 0's literals are visible to the copy
        const uint8_t* src = out + produced - dist;
        for (int i = lane; i < n; i += 32) out[produced + i] = src[i < dist ? i : i % dist];
        __syncwarp();
        produced += n;
        if (produced == limit) return ST_OK;
      }
    }
    if (final) return ST_SHORT;   // produced < limit here
  }
  return status;
}

__global__ void __launch_bounds__(IT) png_inflate_kernel(const uint8_t* __restrict__ files, const int32_t* __restrict__ blocks,
                                                         uint8_t* ws, int H, int W, PngWs L) {
  __shared__ Tables t;
  const int s = blockIdx.x;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const PGeom g = pgeom(blk, H, W);
  const uint8_t* file = files + (size_t)s * L.file;
  uint8_t* base = ws + (size_t)s * L.stride;
  uint8_t* st = base + L.stream;
  // gather the IDAT payloads, each range clamped into the file slot and the total into the stream's room (the slot)
  long long total = 0;
  for (int k = 0; k < g.nidat; ++k) {
    const long long off = min(max((long long)blk[DEFER_PNG_IDAT_OFF + 2 * k], 0ll), (long long)L.slot);
    long long n = min(max((long long)blk[DEFER_PNG_IDAT_OFF + 2 * k + 1], 0ll), (long long)L.slot - off);
    n = min(n, (long long)L.slot - total);
    for (long long i = threadIdx.x; i < n; i += IT) st[total + i] = file[off + i];
    total += n;
  }
  for (int i = threadIdx.x; i < 64; i += IT) st[total + i] = 0;   // bits past the end read as zero
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  long long produced = 0;
  const int status = inflate_warp(t, st, total * 8, base + L.raw, g.raw, produced, lane);
  if (lane == 0) {
    int32_t* stats = reinterpret_cast<int32_t*>(base + L.stats);
    stats[0] = status;
    stats[1] = (int32_t)produced;
    stats[2] = 0;
  }
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : pb <= pc ? b : c;
}

// Unfilter in place: bytes at or past `produced` read as zero (the scanlines the stream did not produce)
__global__ void __launch_bounds__(UT) png_unfilter_kernel(const int32_t* __restrict__ blocks, uint8_t* ws, int H, int W, PngWs L) {
  const int s = blockIdx.x;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const PGeom g = pgeom(blk, H, W);
  uint8_t* base = ws + (size_t)s * L.stride;
  uint8_t* raw = base + L.raw;
  int32_t* stats = reinterpret_cast<int32_t*>(base + L.stats);
  const long long produced = min(max((long long)stats[1], 0ll), g.raw);
  const int bpr = g.bpr, bpp = g.bpp, npx = (bpr + bpp - 1) / bpp;
  const long long rowlen = 1 + (long long)bpr;
  int unknown = 0;
  for (int band = 0; band < g.h; band += UT) {
    const int r = band + threadIdx.x, rows = min(UT, g.h - band);
    const bool active = r < g.h;
    const long long row = (long long)r * rowlen;
    int ft = 0;
    if (active) {
      ft = row < produced ? raw[row] : 0;
      if (ft > 4) {
        ++unknown;
        ft = 0;
      }
    }
    for (int step = 0; step < npx + rows - 1; ++step) {   // row r works on pixel step - (r - band)
      const int x = step - (int)threadIdx.x;
      if (active && x >= 0 && x < npx) {
        for (int b = 0; b < bpp; ++b) {
          const int xb = x * bpp + b;
          if (xb >= bpr) break;
          const long long o = row + 1 + xb;
          const int f = o < produced ? raw[o] : 0;
          const int a = xb >= bpp ? raw[o - bpp] : 0;
          const int u = r > 0 ? raw[o - rowlen] : 0;
          const int c = (r > 0 && xb >= bpp) ? raw[o - rowlen - bpp] : 0;
          const int p = ft == 1 ? a : ft == 2 ? u : ft == 3 ? (a + u) >> 1 : ft == 4 ? paeth(a, u, c) : 0;
          raw[o] = (uint8_t)(f + p);
        }
      }
      __syncthreads();
    }
  }
  if (unknown) atomicAdd(&stats[2], unknown);
}

__device__ __forceinline__ int low_sample(const uint8_t* row, int x, int d) {
  const int bit = x * d;
  return (row[bit >> 3] >> (8 - d - (bit & 7))) & ((1 << d) - 1);
}

__global__ void __launch_bounds__(256) png_expand_kernel(const int32_t* __restrict__ blocks, const uint8_t* __restrict__ ws,
                                                         uint8_t* __restrict__ y_out, int H, int W, PngWs L) {
  const int s = blockIdx.y;
  const int32_t* blk = blocks + (size_t)s * L.block_ints;
  if (!decode_takes(blk, L.take)) return;
  const PGeom g = pgeom(blk, H, W);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.h * g.w) return;
  const int x = i % g.w, r = i / g.w;
  const uint8_t* row = ws + (size_t)s * L.stride + L.raw + (long long)r * (1 + g.bpr) + 1;
  const int d = g.depth;
  int R, G, B;
  if (g.ct == 3) {
    const int idx = d == 8 ? row[x] : low_sample(row, x, d);
    const int v = idx < min(max(blk[8], 0), 256) ? blk[DEFER_PNG_PAL_OFF + idx] : 0;
    R = v & 255;
    G = (v >> 8) & 255;
    B = (v >> 16) & 255;
  } else if (g.ct == 0 || g.ct == 4) {
    const int step = g.ch * (d / 8);
    if (d == 16) R = g.ct == 0 ? min((row[x * step] << 8) | row[x * step + 1], 255) : row[x * step];   // I;16 clips
    else if (d == 8) R = row[x * step];
    else R = low_sample(row, x, d) * (d == 1 ? 255 : d == 2 ? 85 : 17);
    G = B = R;
  } else {   // RGB, RGBA: the high byte at 16 bits
    const int sb = d / 8, p = x * g.ch * sb;
    R = row[p];
    G = row[p + sb];
    B = row[p + 2 * sb];
  }
  uint8_t* o = y_out + (size_t)s * H * W * 3 + (size_t)i * 3;
  o[0] = (uint8_t)R;
  o[1] = (uint8_t)G;
  o[2] = (uint8_t)B;
}

}  // namespace

size_t png_workspace_bytes(int H, int W, int n) { return png_ws(H, W).stride * (size_t)n; }

size_t png_ws_stride(int H, int W, size_t* raw_off) {
  const PngWs L = png_ws(H, W);
  if (raw_off) *raw_off = L.raw;
  return L.stride;
}

// IDAT offsets and lengths in the block are int32: the slot must fit
bool png_bound_ok(int H, int W) { return H >= 1 && W >= 1 && DEFER_PNG_SLOT_BYTES((uint64_t)H, (uint64_t)W) < (1ull << 31); }

int launch_png_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                      cudaStream_t st, const DecodeStrides* strides) {
  PngWs L = png_ws(H, W);
  if (strides) {
    L.file = strides->file;
    L.stride = strides->ws;
    L.block_ints = strides->block_ints;
    L.take = strides->take;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  png_inflate_kernel<<<n, IT, 0, st>>>(files, blocks, ws, H, W, L);
  png_unfilter_kernel<<<n, UT, 0, st>>>(blocks, ws, H, W, L);
  png_expand_kernel<<<dim3((unsigned)(((size_t)H * W + 255) / 256), (unsigned)n), 256, 0, st>>>(blocks, ws, y, H, W, L);
  DEFER_CUDA(cudaGetLastError());
  return DEFER_OK;
}

}  // namespace defer

using namespace defer;

extern "C" {

int defer_k_png_workspace(int H, int W, int n, uint64_t* bytes, uint64_t* sample_stride, uint64_t* raw_off) {
  DEFER_CHECK(n >= 1 && png_bound_ok(H, W), "k_png_workspace: bad bound %dx%d (n %d)", H, W, n);
  const PngWs L = png_ws(H, W);
  if (bytes) *bytes = L.stride * (uint64_t)n;
  if (sample_stride) *sample_stride = L.stride;
  if (raw_off) *raw_off = L.raw;
  return DEFER_OK;
}

int defer_k_png_decode(const uint8_t* files, const int32_t* blocks, int n, int H, int W, void* workspace, uint8_t* y,
                       void* stream) {
  DEFER_CHECK(files && blocks && workspace && y, "k_png_decode: null pointer");
  DEFER_CHECK(n >= 1 && n <= 65535 && png_bound_ok(H, W), "k_png_decode: bad sizes (n %d, bound %dx%d)", n, H, W);
  DEFER_CHECK(((uintptr_t)blocks & 3) == 0 && ((uintptr_t)workspace & 255) == 0,
              "k_png_decode: blocks must be 4-byte and the workspace 256-byte aligned");
  return launch_png_decode(files, blocks, n, H, W, workspace, y, (cudaStream_t)stream);
}

}  // extern "C"
