// Baseline JPEG decode on the device (SURVEY.md section 8f rank 2), equal bit for bit to what PIL's libjpeg-turbo gives with
// its defaults (islow IDCT, fancy upsampling, jdcolor.c's fixed-point YCbCr -> RGB), as restated in oracle/jpeg_ref.py.
//
// Scope: SOF0 / SOF1, 8-bit, Huffman, one scan holding every component; 3-component YCbCr with luma h1v1 / h2v1 / h1v2 / h2v2
// and chroma 1x1, or 1-component gray; optional restart intervals.  Everything else is refused by the host parse before
// anything is uploaded.
//
// Pipeline (one launch per stage over the whole batch; blockIdx.y = image):
//   k_jpeg_markers   end of the scan = the first marker that is not RSTn
//   k_jpeg_count     per 4 KiB tile: data bytes (0xFF 0x00 -> 0xFF, markers and fill bytes dropped) and RST markers
//   k_jpeg_tiles     per image: exclusive scan of the tile counts
//   k_jpeg_compact   write the unstuffed bytes and the byte position where every restart interval starts
//   k_jpeg_sync_chunk self-synchronising Huffman decode (Klein & Wiseman 2003; Weissenberger & Schmidt, ICPP 2018): the
//                    unstuffed bits are cut into JPEG_SUB-bit subsequences and each CTA takes JPEG_CHUNK of them.  Every
//                    thread decodes from a guessed state (its subsequence's first bit, block 0 of an MCU, DC next) and goes
//                    on, one subsequence per lock-step iteration, until its path merges with the path started one
//                    subsequence later; the chunk then holds one path from its first subsequence's guess.
//   k_jpeg_sync_round  rounds over chunks: each chunk re-decodes from the previous chunk's last exit until it meets its
//                    recorded path; the rounds stop once one changes nothing.  Restart intervals begin in a known state,
//                    so a decode that reaches one is synchronised.
//   k_jpeg_sync_serial  images still changing after JPEG_ROUNDS rounds: one thread chains every exit state in order (slow,
//                    always right)
//   k_jpeg_bases     per image: exclusive scan of the per-subsequence block counts
//   k_jpeg_write     decode again from the confirmed entry states and write the quantised coefficients, int16, MCU order
//   k_jpeg_dc        per component: DC differences -> values, a segmented scan that restarts with every restart interval
//   k_jpeg_idct      dequantise + islow IDCT into component planes
//   k_jpeg_color     fancy upsampling + YCbCr -> RGB into the caller's H x W x 3 buffers
// Every read of the stream is bounded by the scan length; an invalid code, a coefficient index past 63, a wrong MCU count or
// a restart marker out of sequence sets the image's status and nothing else.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int JPEG_TILE = 4096;        // bytes per tile of the byte passes (256 threads x 16)
constexpr int JPEG_SUB = 1024;         // bits per subsequence
constexpr int JPEG_ROUNDS = 8;         // synchronisation rounds before the serial chain
constexpr int JPEG_CHUNK = 256;        // subsequences synchronised together by one CTA
constexpr int JPEG_MAX_BATCH = 256;
constexpr int JPEG_MAX_SIDE = 16384;
constexpr int64_t JPEG_MAX_PIXELS = int64_t(1) << 26;
constexpr size_t JPEG_MAX_BYTES = size_t(1) << 28;  // per file: bit positions stay below 2^31

// status codes (include/gtsfm_b200.h)
constexpr int J_LIMIT = -2, J_HEADER = -10, J_PROGRESSIVE = -11, J_ARITH = -12, J_LOSSLESS = -13, J_PRECISION = -14,
              J_COMPONENTS = -15, J_RGB = -16, J_SAMPLING = -17, J_MULTISCAN = -18, J_DNL = -19, J_TRUNCATED = -20,
              J_CORRUPT = -21, J_HUFFTABLE = -22;

struct JpegHuff {
  uint16_t lut[512];    // 9-bit lookahead: (length << 8) | symbol, 0 = longer than 9 bits (or invalid)
  int32_t maxcode[17];  // largest code of each length (-1: none)
  int32_t valoff[17];   // symbol index = code + valoff[length]
  uint8_t vals[256];
};

struct JpegImg {  // per image, uploaded with the batch; the last fields are written on the device
  uint64_t in_off;  // offset of the scan's first byte in the byte buffer (a tile multiple); the unstuffed bytes go to the same offset
  uint32_t in_len;  // bytes from the scan's first byte to the end of the file
  uint32_t tile0;   // first tile in the tile arrays
  uint32_t sub0, nsub_cap;  // subsequence slots
  uint32_t rst0, nseg;      // restart slots (nseg - 1 used), intervals
  int width, height, ncomp, hmax, vmax, mcux, mcuy, bpm, ri;  // ri = MCUs per restart interval (all MCUs when there is no DRI)
  int hs[3], vs[3], boff[3];  // blocks per MCU of each component, first block of the component within the MCU
  int pw[3], ph[3];           // plane width / height (MCU-padded); cw / ch = downsampled size
  int cw[3], ch[3];
  uint64_t coef_off;  // first block in the coefficient buffer
  uint64_t plane_off[3];
  uint32_t nblocks;
  uint32_t huff;     // index of this image's first JpegHuff (dc0 dc1 dc2 ac0 ac1 ac2)
  uint16_t q[3][64];  // quantisation tables per component, natural order
  uint8_t* out;
  uint64_t out_pitch;
  // device-written
  uint32_t end;    // first byte of the terminating marker (initialised to in_len)
  uint32_t len;    // unstuffed bytes
  uint32_t nrst;
  int status;
  int rounds;
};

__device__ __constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                                41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                                30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- host parse ---------------------------------------------------------------------------------------------------------
struct HostComp {
  int id, h, v, tq, td, ta;
};
struct HostHeader {
  int width = 0, height = 0, ncomp = 0, restart = 0;
  HostComp c[3];
  size_t scan_off = 0;
  const uint8_t* qt[4] = {};  // raw DQT payload (zig-zag order)
  int qprec[4] = {};
  const uint8_t* ht[2][4] = {};  // raw DHT payload: 16 counts then symbols
};

int check_huffman(const uint8_t* t, bool dc) {
  int code = 0, total = 0;
  for (int l = 1; l <= 16; ++l) {
    code += t[l - 1];
    total += t[l - 1];
    if (code > (1 << l)) return J_HEADER;
    if (t[l - 1] && code == (1 << l)) return J_HUFFTABLE;  // an all-ones code: never written by encoders (T.81 Annex C)
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < total; ++i)
      if (t[16 + i] > 15) return J_HEADER;
  return 0;
}

bool has_eoi(const uint8_t* d, size_t n, size_t from) {
  for (size_t p = n; p >= from + 2; --p)
    if (d[p - 2] == 0xFF && d[p - 1] == 0xD9) return true;
  return false;
}

int parse_header(const uint8_t* d, size_t n, HostHeader& hd) {
  if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) return J_HEADER;
  if (n > JPEG_MAX_BYTES) return J_LIMIT;
  size_t p = 2;
  bool frame = false, jfif = false;
  int adobe = -1;
  while (true) {
    while (p + 1 < n && d[p] == 0xFF && d[p + 1] == 0xFF) ++p;
    if (p + 4 > n || d[p] != 0xFF) return J_HEADER;
    const int m = d[p + 1];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return J_HEADER;
    const size_t len = (size_t(d[p + 2]) << 8) | d[p + 3];
    if (len < 2 || p + 2 + len > n) return J_HEADER;
    const uint8_t* s = d + p + 4;
    const size_t sl = len - 2;
    p += 2 + len;
    if (m == 0xC0 || m == 0xC1) {
      if (frame || sl < 6) return J_HEADER;
      if (s[0] != 8) return J_PRECISION;
      hd.height = (s[1] << 8) | s[2];
      hd.width = (s[3] << 8) | s[4];
      hd.ncomp = s[5];
      if (hd.height == 0) return J_DNL;
      if (hd.width == 0 || sl < size_t(6 + 3 * hd.ncomp)) return J_HEADER;
      if (hd.ncomp != 1 && hd.ncomp != 3) return J_COMPONENTS;
      for (int i = 0; i < hd.ncomp; ++i) hd.c[i] = {s[6 + 3 * i], s[7 + 3 * i] >> 4, s[7 + 3 * i] & 15, s[8 + 3 * i], 0, 0};
      frame = true;
    } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
      return J_PROGRESSIVE;
    } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF || m == 0xC5) {
      return J_LOSSLESS;
    } else if (m == 0xC9 || m == 0xCD || m == 0xCC) {
      return J_ARITH;
    } else if (m == 0xC4) {
      size_t q = 0;
      while (q < sl) {
        if (q + 17 > sl) return J_HEADER;
        const int tc = s[q] >> 4, th = s[q] & 15;
        int cnt = 0;
        for (int l = 0; l < 16; ++l) cnt += s[q + 1 + l];
        if (tc > 1 || th > 3 || cnt > 256 || q + 17 + cnt > sl) return J_HEADER;
        const int rc = check_huffman(s + q + 1, tc == 0);
        if (rc) return rc;
        hd.ht[tc][th] = s + q + 1;
        q += 17 + cnt;
      }
    } else if (m == 0xDB) {
      size_t q = 0;
      while (q < sl) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        if (pq > 1 || tq > 3 || q + 1 + 64 * (pq + 1) > sl) return J_HEADER;
        hd.qt[tq] = s + q + 1;
        hd.qprec[tq] = pq;
        q += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (sl < 2) return J_HEADER;
      hd.restart = (s[0] << 8) | s[1];
    } else if (m == 0xE0) {
      if (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;  // libjpeg's examine_app0 needs 14 bytes
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = s[11];
    } else if (m == 0xDA) {
      if (!frame || sl < 1) return J_HEADER;
      const int ns = s[0];
      if (sl < size_t(4 + 2 * ns)) return J_HEADER;
      if (ns != hd.ncomp) return J_MULTISCAN;
      for (int i = 0; i < ns; ++i) {
        if (s[1 + 2 * i] != hd.c[i].id) return J_MULTISCAN;  // scan order differs from the frame
        hd.c[i].td = s[2 + 2 * i] >> 4;
        hd.c[i].ta = s[2 + 2 * i] & 15;
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return J_HEADER;
      if (hd.ncomp == 3 && !jfif) {  // libjpeg's colour-space guess (jdapimin.c default_decompress_parms)
        if (adobe == 0) return J_RGB;
        if (adobe < 0 && hd.c[0].id == 82 && hd.c[1].id == 71 && hd.c[2].id == 66) return J_RGB;
      }
      if (hd.ncomp == 1) {
        if (hd.c[0].h < 1 || hd.c[0].h > 4 || hd.c[0].v < 1 || hd.c[0].v > 4) return J_HEADER;
      } else {
        const int h = hd.c[0].h, v = hd.c[0].v;
        if (h < 1 || h > 2 || v < 1 || v > 2) return J_SAMPLING;
        for (int i = 1; i < 3; ++i)
          if (hd.c[i].h != 1 || hd.c[i].v != 1) return J_SAMPLING;
      }
      for (int i = 0; i < hd.ncomp; ++i)
        if (hd.c[i].tq > 3 || !hd.qt[hd.c[i].tq] || hd.c[i].td > 3 || !hd.ht[0][hd.c[i].td] || hd.c[i].ta > 3 || !hd.ht[1][hd.c[i].ta])
          return J_HEADER;
      if (!has_eoi(d, n, p)) return J_TRUNCATED;
      if (hd.width > JPEG_MAX_SIDE || hd.height > JPEG_MAX_SIDE || int64_t(hd.width) * hd.height > JPEG_MAX_PIXELS) return J_LIMIT;
      hd.scan_off = p;
      return 0;
    }
    // APPn, COM and other segments with a length: skipped
  }
}

void build_huff(const uint8_t* t, JpegHuff& h) {
  memset(&h, 0, sizeof(h));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int cnt = t[l - 1];
    h.valoff[l] = k - code;
    h.maxcode[l] = cnt ? code + cnt - 1 : -1;
    for (int i = 0; i < cnt; ++i, ++k, ++code) {
      h.vals[k] = t[16 + k];
      if (l <= 9)
        for (int f = 0; f < (1 << (9 - l)); ++f) h.lut[(code << (9 - l)) | f] = uint16_t((l << 8) | t[16 + k]);
    }
    code <<= 1;
  }
}

// ---- device helpers ----------------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t* s;
  uint32_t nbytes, next;
  uint64_t buf;
  int cnt;
  __device__ void seek(uint32_t pos) {
    next = pos >> 3;
    buf = 0;
    cnt = 0;
    refill();
    buf <<= (pos & 7);
    cnt -= (pos & 7);
  }
  __device__ void refill() {
    while (cnt <= 56) {
      const uint64_t b = next < nbytes ? __ldg(s + next) : 0;
      buf |= b << (56 - cnt);
      cnt += 8;
      ++next;
    }
  }
  __device__ uint32_t peek16() const { return uint32_t(buf >> 48); }
  __device__ void skip(int n) {
    buf <<= n;
    cnt -= n;
    if (cnt < 32) refill();
  }
};

// one Huffman symbol from the 16 bits `w`: symbol, *len = code length; -1 = no code
__device__ __forceinline__ int huff_decode(const JpegHuff* __restrict__ t, uint32_t w, int* len) {
  const uint32_t e = t->lut[w >> 7];
  if (e) {
    *len = int(e >> 8);
    return int(e & 255);
  }
  for (int l = 10; l <= 16; ++l) {
    const int code = int(w >> (16 - l));
    if (code <= t->maxcode[l]) {
      *len = l;
      return t->vals[code + t->valoff[l]];
    }
  }
  return -1;
}

__device__ __forceinline__ int huff_extend(uint32_t v, int s) { return v < (1u << (s - 1)) ? int(v) - (1 << s) + 1 : int(v); }

// packed decoder state: bit position | block within the MCU << 32 | zig-zag index (0 = DC next) << 36 | DC symbols << 44
constexpr uint64_t J_ERR_STATE = ~uint64_t(0);
constexpr uint64_t J_PHASE_MASK = (uint64_t(1) << 44) - 1;
__device__ __forceinline__ uint64_t pack_state(uint32_t pos, int b, int z, int count) {
  return uint64_t(pos) | (uint64_t(b) << 32) | (uint64_t(z) << 36) | (uint64_t(count) << 44);
}

struct Dec {
  const uint8_t* s;
  uint32_t nbits;
  const uint32_t* rst;  // byte position of every interval start after the first
  int nseg;
  const JpegHuff* huff;  // dc0 dc1 dc2 ac0 ac1 ac2
  int boff1, boff2;      // first block of components 1 and 2 within the MCU
  int bpm;
};

__device__ __forceinline__ uint32_t seg_start(const Dec& d, int k) { return k == 0 ? 0u : 8u * d.rst[k - 1]; }
__device__ __forceinline__ uint32_t seg_end(const Dec& d, int k) { return k + 1 >= d.nseg ? d.nbits : 8u * d.rst[k]; }

__device__ int seg_of(const Dec& d, uint32_t pos) {  // last interval starting at or before pos
  int lo = 0, hi = d.nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg_start(d, mid) <= pos) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct Writer {
  int16_t* coef;  // the image's blocks
  int64_t blk;    // block being written
  uint32_t nblocks;
  int ri, bpm, mcus;
  bool bad;
};

// Decode from (pos, b, z) to the first symbol boundary at or past sub_end (oracle/jpeg_ref.py `_f`).  At the end of a restart
// interval (an MCU boundary followed by fewer than 8 one bits up to the interval's end) decoding continues from the next
// interval's start.  While synchronising, a decode error restarts the guess there (or at the next bit in the last interval);
// with a Writer it marks the image corrupt instead.
template <bool WRITE>
__device__ uint64_t jpeg_walk(const Dec& d, uint32_t pos, int b, int z, uint32_t sub_end, Writer* w) {
  int count = 0;
  pos = min(pos, d.nbits);
  int seg = seg_of(d, pos);
  uint32_t end = seg_end(d, seg);
  BitReader br;
  br.s = d.s;
  br.nbytes = (d.nbits + 7) >> 3;
  br.seek(pos);
  while (true) {
    if (b == 0 && z == 0 && end - pos < 8) {
      const int r = int(end - pos);
      if (r == 0 || (br.peek16() >> (16 - r)) == (1u << r) - 1) {  // interval done
        if (WRITE) {
          const int64_t want = int64_t(min((seg + 1) * w->ri, w->mcus)) * w->bpm;
          if (w->blk + 1 != want) w->bad = true;
        }
        if (seg + 1 >= d.nseg) return pack_state(end, 0, 0, count);
        ++seg;
        pos = seg_start(d, seg);
        end = seg_end(d, seg);
        br.seek(pos);
        if (pos >= sub_end) return pack_state(pos, 0, 0, count);
        continue;
      }
    }
    if (pos >= sub_end) return pack_state(pos, b, z, count);
    const int ci = b < d.boff1 ? 0 : (b < d.boff2 ? 1 : 2);
    bool ok = true;
    int len;
    const uint32_t w16 = br.peek16();
    if (z == 0) {
      const int s = huff_decode(d.huff + ci, w16, &len);
      if (s < 0 || pos + len + s > end) {
        ok = false;
      } else {
        br.skip(len);
        int v = 0;
        if (s) {
          v = huff_extend(br.peek16() >> (16 - s), s);
          br.skip(s);
        }
        pos += len + s;
        ++count;
        z = 1;
        if (WRITE) {
          ++w->blk;
          if (w->blk >= w->nblocks) w->bad = true;
          else w->coef[w->blk * 64] = int16_t(v);
        }
      }
    } else {
      const int rs = huff_decode(d.huff + 3 + ci, w16, &len);
      const int run = rs >> 4, s = rs & 15;
      if (rs < 0 || pos + len + s > end) {
        ok = false;
      } else if (s) {
        const int k = z + run;
        if (k > 63) {
          ok = false;
        } else {
          br.skip(len);
          const int v = huff_extend(br.peek16() >> (16 - s), s);
          br.skip(s);
          pos += len + s;
          if (WRITE && w->blk >= 0 && w->blk < w->nblocks) {
            int16_t* c = w->coef + w->blk * 64;
            for (int i = z; i < k; ++i) c[c_zigzag[i]] = 0;
            c[c_zigzag[k]] = int16_t(v);
          }
          z = k + 1;
        }
      } else {
        const int zn = run == 15 ? z + 16 : 64;  // ZRL or EOB
        if (zn > 64) {
          ok = false;
        } else {
          br.skip(len);
          pos += len;
          if (WRITE && w->blk >= 0 && w->blk < w->nblocks) {
            int16_t* c = w->coef + w->blk * 64;
            for (int i = z; i < zn; ++i) c[c_zigzag[i]] = 0;
          }
          z = zn;
        }
      }
    }
    if (!ok) {
      if (WRITE) {
        w->bad = true;
        return J_ERR_STATE;
      }
      // while synchronising, an error only means a wrong guess: guess again from the next restart interval, or from the
      // next bit when this is the last interval (a path that gave up here could never merge with the true one)
      b = 0;
      z = 0;
      if (seg + 1 < d.nseg) {
        ++seg;
        pos = seg_start(d, seg);
        end = seg_end(d, seg);
      } else {
        ++pos;
      }
      br.seek(pos);
      if (pos >= sub_end) return pack_state(pos, 0, 0, count);
      continue;
    }
    if (z == 64) {
      z = 0;
      if (++b == d.bpm) b = 0;
    }
  }
}

__device__ Dec make_dec(const JpegImg& im, const uint8_t* un, const uint32_t* rst, const JpegHuff* huff) {
  Dec d;
  d.s = un + im.in_off;
  d.nbits = 8u * im.len;
  d.rst = rst + im.rst0;
  d.nseg = int(im.nseg);
  d.huff = huff + im.huff;
  d.boff1 = im.ncomp > 1 ? im.boff[1] : im.bpm;
  d.boff2 = im.ncomp > 2 ? im.boff[2] : im.bpm;
  d.bpm = im.bpm;
  return d;
}

__device__ __forceinline__ uint32_t nsub_of(const JpegImg& im) {
  return min(max(1u, (8u * im.len + JPEG_SUB - 1) / JPEG_SUB), im.nsub_cap);
}

// block-wide exclusive scan (blockDim.x a multiple of 32, at most 1024); `total` = the block's sum
template <typename T>
__device__ T block_scan_excl(T v, T* sh, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    T s = lane < nw ? sh[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sh[lane] = s;
  }
  __syncthreads();
  const T pre = warp ? sh[warp - 1] : T(0);
  total = sh[nw - 1];
  __syncthreads();
  return pre + x - v;
}

// ---- byte passes -------------------------------------------------------------------------------------------------------
__global__ void k_jpeg_markers(JpegImg* __restrict__ imgs, const uint8_t* __restrict__ in) {
  JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  const uint8_t* s = in + im.in_off;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < im.in_len; p += gridDim.x * blockDim.x) {
    if (s[p] != 0xFF) continue;
    const int nx = p + 1 < im.in_len ? s[p + 1] : -1;
    if (nx != 0x00 && nx != 0xFF && !(nx >= 0xD0 && nx <= 0xD7)) atomicMin(&im.end, p);
  }
}

// classification of byte p < end: 1 = data byte, 2 = restart marker code, 0 = dropped
__device__ __forceinline__ int jpeg_byte_class(const uint8_t* s, uint32_t p, uint32_t n) {
  const uint8_t b = s[p];
  if (b == 0xFF) return (p + 1 < n && s[p + 1] == 0x00) ? 1 : 0;
  if (p > 0 && s[p - 1] == 0xFF) return (b >= 0xD0 && b <= 0xD7) ? 2 : 0;
  return 1;
}

__global__ void __launch_bounds__(256) k_jpeg_count(const JpegImg* __restrict__ imgs, const uint8_t* __restrict__ in, uint64_t* __restrict__ tile_cnt) {
  const JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  __shared__ uint64_t sh[32];
  const uint8_t* s = in + im.in_off;
  const uint32_t ntiles = (im.in_len + JPEG_TILE - 1) / JPEG_TILE;
  for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    uint64_t c = 0;  // data bytes | restart markers << 32
    const uint32_t p0 = t * JPEG_TILE + threadIdx.x * 16;
    for (int i = 0; i < 16; ++i) {
      const uint32_t p = p0 + i;
      if (p >= im.end) break;
      const int k = jpeg_byte_class(s, p, im.in_len);
      c += k == 1 ? 1ull : (k == 2 ? (1ull << 32) : 0ull);
    }
    uint64_t tot;
    block_scan_excl<uint64_t>(c, sh, tot);
    if (threadIdx.x == 0) tile_cnt[im.tile0 + t] = tot;
  }
}

__global__ void __launch_bounds__(1024) k_jpeg_tiles(JpegImg* __restrict__ imgs, uint64_t* __restrict__ tile_cnt) {
  JpegImg& im = imgs[blockIdx.x];
  if (im.status) return;
  __shared__ uint64_t sh[32];
  const uint32_t ntiles = (im.in_len + JPEG_TILE - 1) / JPEG_TILE;
  uint64_t carry = 0;
  for (uint32_t t0 = 0; t0 < ntiles; t0 += blockDim.x) {
    const uint32_t t = t0 + threadIdx.x;
    const uint64_t v = t < ntiles ? tile_cnt[im.tile0 + t] : 0;
    uint64_t tot;
    const uint64_t ex = block_scan_excl<uint64_t>(v, sh, tot);
    if (t < ntiles) tile_cnt[im.tile0 + t] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    im.len = uint32_t(carry);
    im.nrst = uint32_t(carry >> 32);
    if (im.nrst + 1 != im.nseg) im.status = J_CORRUPT;
  }
}

__global__ void __launch_bounds__(256) k_jpeg_compact(JpegImg* __restrict__ imgs, const uint8_t* __restrict__ in, const uint64_t* __restrict__ tile_pre,
                                                       uint8_t* __restrict__ un, uint32_t* __restrict__ rst) {
  JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  __shared__ uint64_t sh[32];
  const uint8_t* s = in + im.in_off;
  uint8_t* o = un + im.in_off;
  const uint32_t ntiles = (im.in_len + JPEG_TILE - 1) / JPEG_TILE;
  for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const uint32_t p0 = t * JPEG_TILE + threadIdx.x * 16;
    uint64_t c = 0;
    for (int i = 0; i < 16; ++i) {
      const uint32_t p = p0 + i;
      if (p >= im.end) break;
      const int k = jpeg_byte_class(s, p, im.in_len);
      c += k == 1 ? 1ull : (k == 2 ? (1ull << 32) : 0ull);
    }
    uint64_t tot;
    uint64_t pre = tile_pre[im.tile0 + t] + block_scan_excl<uint64_t>(c, sh, tot);
    for (int i = 0; i < 16; ++i) {
      const uint32_t p = p0 + i;
      if (p >= im.end) break;
      const int k = jpeg_byte_class(s, p, im.in_len);
      if (k == 1) {
        o[uint32_t(pre)] = s[p];
        pre += 1;
      } else if (k == 2) {
        const uint32_t r = uint32_t(pre >> 32);
        if (r + 1 < im.nseg) {
          rst[im.rst0 + r] = uint32_t(pre);
          if (s[p] != 0xD0 + (r & 7)) im.status = J_CORRUPT;  // out of sequence
        }
        pre += 1ull << 32;
      }
    }
  }
}

// ---- entropy decode ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t walk_from(const Dec& d, uint64_t e, uint32_t sub_end) {
  return e == J_ERR_STATE ? J_ERR_STATE : jpeg_walk<false>(d, uint32_t(e), int((e >> 32) & 15), int((e >> 36) & 127), sub_end, nullptr);
}

// One CTA per chunk of JPEG_CHUNK subsequences.  Thread t starts at subsequence c0 + t from the guessed state and, in lock step
// with the others, decodes one subsequence further per iteration.  In iteration i it decodes subsequence c0 + t + i, whose
// recorded exit was written one iteration earlier by the path that started one subsequence later; once its exit agrees with
// that one in (position, block, coefficient index) the two paths have merged and the thread stops.  The lowest path still
// running writes each slot last, so afterwards the chunk holds the decode from its first subsequence's guessed state.
__global__ void __launch_bounds__(JPEG_CHUNK) k_jpeg_sync_chunk(const JpegImg* __restrict__ imgs, const uint8_t* __restrict__ un,
                                                                const uint32_t* __restrict__ rst, const JpegHuff* __restrict__ huff,
                                                                uint64_t* __restrict__ exits) {
  const JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  const uint32_t nsub = nsub_of(im);
  const Dec d = make_dec(im, un, rst, huff);
  uint64_t* ex = exits + im.sub0;
  for (uint32_t c0 = blockIdx.x * JPEG_CHUNK; c0 < nsub; c0 += gridDim.x * JPEG_CHUNK) {
    const uint32_t c1 = min(c0 + uint32_t(JPEG_CHUNK), nsub);
    uint32_t k = c0 + threadIdx.x;
    bool active = k < c1, first = true;
    uint64_t st = pack_state(k * uint32_t(JPEG_SUB), 0, 0, 0);
    while (__syncthreads_or(active)) {
      uint64_t v = 0, old = 0;
      if (active) {
        v = walk_from(d, st, min((k + 1) * uint32_t(JPEG_SUB), d.nbits));
        old = ex[k];
      }
      __syncthreads();
      if (active) {
        ex[k] = v;
        // the next subsequence depends on (position, block, coefficient index) only, not on this one's block count
        if (!first && (v & J_PHASE_MASK) == (old & J_PHASE_MASK)) active = false;
        first = false;
        st = v;
        if (++k >= c1) active = false;
      }
    }
  }
}

// Round r >= 1, while the previous round changed something: one thread per chunk after the first re-decodes from the exit
// of the chunk before it, writing its chunk's exits until they merge with the recorded path.  A round that writes nothing
// leaves every exit equal to the decode of its subsequence from its predecessor's exit, i.e. the sequential decode.
__global__ void __launch_bounds__(128) k_jpeg_sync_round(JpegImg* __restrict__ imgs, const uint8_t* __restrict__ un, const uint32_t* __restrict__ rst,
                                                          const JpegHuff* __restrict__ huff, uint64_t* __restrict__ exits,
                                                          int* __restrict__ changed, int round, int n_images) {
  JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  if (round >= 2 && !changed[(round - 1) * n_images + blockIdx.y]) return;
  const uint32_t nsub = nsub_of(im), nchunks = (nsub + JPEG_CHUNK - 1) / JPEG_CHUNK;
  const Dec d = make_dec(im, un, rst, huff);
  volatile uint64_t* ex = exits + im.sub0;
  for (uint32_t c = 1 + blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += gridDim.x * blockDim.x) {
    const uint32_t c0 = c * JPEG_CHUNK, c1 = min(c0 + uint32_t(JPEG_CHUNK), nsub);
    uint64_t e = ex[c0 - 1];  // old or new value of this round: either is a valid iterate
    for (uint32_t k = c0; k < c1; ++k) {
      const uint64_t v = walk_from(d, e, min((k + 1) * uint32_t(JPEG_SUB), d.nbits));
      const uint64_t old = ex[k];
      if (v == old) break;
      ex[k] = v;
      changed[round * n_images + blockIdx.y] = 1;
      if ((v & J_PHASE_MASK) == (old & J_PHASE_MASK)) break;
      e = v;
    }
  }
}

__global__ void k_jpeg_sync_serial(JpegImg* __restrict__ imgs, const uint8_t* __restrict__ un, const uint32_t* __restrict__ rst,
                                   const JpegHuff* __restrict__ huff, uint64_t* __restrict__ exits, const int* __restrict__ changed, int n_images) {
  JpegImg& im = imgs[blockIdx.x];
  if (im.status || threadIdx.x != 0) return;
  int r = 1;
  while (r <= JPEG_ROUNDS && changed[r * n_images + blockIdx.x]) ++r;
  im.rounds = r;
  if (r <= JPEG_ROUNDS) return;
  const uint32_t nsub = nsub_of(im);
  const Dec d = make_dec(im, un, rst, huff);
  uint64_t* ex = exits + im.sub0;
  for (uint32_t j = 1; j < nsub; ++j) {
    const uint64_t e = ex[j - 1];
    const uint32_t sub_end = min((j + 1) * uint32_t(JPEG_SUB), d.nbits);
    ex[j] = e == J_ERR_STATE ? J_ERR_STATE : jpeg_walk<false>(d, uint32_t(e), int((e >> 32) & 15), int((e >> 36) & 127), sub_end, nullptr);
  }
}

__global__ void __launch_bounds__(1024) k_jpeg_bases(JpegImg* __restrict__ imgs, const uint64_t* __restrict__ exits, uint32_t* __restrict__ bases) {
  JpegImg& im = imgs[blockIdx.x];
  if (im.status) return;
  __shared__ uint32_t sh[32];
  const uint32_t nsub = nsub_of(im);
  const uint64_t* ex = exits + im.sub0;
  uint32_t carry = 0;
  bool err = false;
  for (uint32_t j0 = 0; j0 < nsub; j0 += blockDim.x) {
    const uint32_t j = j0 + threadIdx.x;
    uint32_t c = 0;
    if (j < nsub) {
      if (ex[j] == J_ERR_STATE) err = true;
      else c = uint32_t(ex[j] >> 44);
    }
    uint32_t tot;
    const uint32_t pre = block_scan_excl<uint32_t>(c, sh, tot);
    if (j < nsub) bases[im.sub0 + j] = carry + pre;
    carry += tot;
  }
  err = __syncthreads_or(err);
  if (threadIdx.x == 0) {
    const uint64_t last = ex[nsub - 1];
    if (err || carry != im.nblocks || uint32_t(last) != 8u * im.len || ((last >> 32) & 0x7ff) != 0) im.status = J_CORRUPT;
  }
}

__global__ void __launch_bounds__(128) k_jpeg_write(JpegImg* __restrict__ imgs, const uint8_t* __restrict__ un, const uint32_t* __restrict__ rst,
                                                     const JpegHuff* __restrict__ huff, const uint64_t* __restrict__ exits,
                                                     const uint32_t* __restrict__ bases, int16_t* __restrict__ coef) {
  JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  const uint32_t nsub = nsub_of(im);
  const Dec d = make_dec(im, un, rst, huff);
  const uint64_t* ex = exits + im.sub0;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nsub; j += gridDim.x * blockDim.x) {
    const uint64_t e = j ? ex[j - 1] : 0;
    Writer w{coef + im.coef_off * 64, int64_t(bases[im.sub0 + j]) - 1, im.nblocks, im.ri, im.bpm, im.mcux * im.mcuy, false};
    const uint32_t sub_end = min((j + 1) * uint32_t(JPEG_SUB), d.nbits);
    const uint64_t v = jpeg_walk<true>(d, uint32_t(e), int((e >> 32) & 15), int((e >> 36) & 127), sub_end, &w);
    if (w.bad || v != ex[j]) im.status = J_CORRUPT;
  }
}

// DC differences -> values: per (image, component) a scan over the component's blocks in MCU order that restarts with
// every restart interval (int accumulation, stored as int16 like libjpeg's JCOEF)
__global__ void __launch_bounds__(1024) k_jpeg_dc(const JpegImg* __restrict__ imgs, int16_t* __restrict__ coef) {
  const JpegImg& im = imgs[blockIdx.y];
  const int c = blockIdx.x;
  if (im.status || c >= im.ncomp) return;
  __shared__ int s_sum[1024];
  __shared__ int s_flag[1024];
  const int per = im.hs[c] * im.vs[c];
  const int64_t nc = int64_t(im.mcux) * im.mcuy * per;
  const int64_t chunk = (nc + blockDim.x - 1) / blockDim.x;
  const int64_t k0 = threadIdx.x * chunk, k1 = min(nc, k0 + chunk);
  int16_t* cf = coef + im.coef_off * 64;
  auto idx = [&](int64_t k) { const int64_t m = k / per; return (m * im.bpm + im.boff[c] + (k - m * per)) * 64; };
  auto reset = [&](int64_t k) { const int64_t m = k / per; return (k - m * per) == 0 && (m % im.ri) == 0; };
  int sum = 0, flag = 0;
  for (int64_t k = k0; k < k1; ++k) {
    if (reset(k)) {
      sum = 0;
      flag = 1;
    }
    sum += cf[idx(k)];
  }
  s_sum[threadIdx.x] = sum;
  s_flag[threadIdx.x] = flag;
  __syncthreads();
  for (int o = 1; o < (int)blockDim.x; o <<= 1) {  // inclusive segmented scan (Hillis-Steele)
    int ps = 0, pf = 0;
    if ((int)threadIdx.x >= o) {
      ps = s_sum[threadIdx.x - o];
      pf = s_flag[threadIdx.x - o];
    }
    __syncthreads();
    if ((int)threadIdx.x >= o && !s_flag[threadIdx.x]) {
      s_sum[threadIdx.x] += ps;
      s_flag[threadIdx.x] = pf;
    }
    __syncthreads();
  }
  int run = threadIdx.x ? s_sum[threadIdx.x - 1] : 0;
  for (int64_t k = k0; k < k1; ++k) {
    if (reset(k)) run = 0;
    const int64_t i = idx(k);
    run += cf[i];
    cf[i] = int16_t(run);
  }
}

// ---- reconstruction ----------------------------------------------------------------------------------------------------
#define J_FIX_0_298 2446
#define J_FIX_0_390 3196
#define J_FIX_0_541 4433
#define J_FIX_0_765 6270
#define J_FIX_0_899 7373
#define J_FIX_1_175 9633
#define J_FIX_1_501 12299
#define J_FIX_1_847 15137
#define J_FIX_1_961 16069
#define J_FIX_2_053 16819
#define J_FIX_2_562 20995
#define J_FIX_3_072 25172

// libjpeg-turbo's jpeg_idct_islow butterfly (CONST_BITS 13, PASS1_BITS 2) on one column / row
__device__ __forceinline__ void idct_1d(int s0, int s1, int s2, int s3, int s4, int s5, int s6, int s7, int out[8]) {
  int z1 = (s2 + s6) * J_FIX_0_541;
  const int tmp2 = z1 + s6 * -J_FIX_1_847;
  const int tmp3 = z1 + s2 * J_FIX_0_765;
  const int tmp0 = (s0 + s4) * 8192;
  const int tmp1 = (s0 - s4) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int o0 = s7, o1 = s5, o2 = s3, o3 = s1;
  z1 = o0 + o3;
  int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const int z5 = (z3 + z4) * J_FIX_1_175;
  o0 *= J_FIX_0_298;
  o1 *= J_FIX_2_053;
  o2 *= J_FIX_3_072;
  o3 *= J_FIX_1_501;
  z1 *= -J_FIX_0_899;
  z2 *= -J_FIX_2_562;
  z3 = z3 * -J_FIX_1_961 + z5;
  z4 = z4 * -J_FIX_0_390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  out[0] = t10 + o3;
  out[7] = t10 - o3;
  out[1] = t11 + o2;
  out[6] = t11 - o2;
  out[2] = t12 + o1;
  out[5] = t12 - o1;
  out[3] = t13 + o0;
  out[4] = t13 - o0;
}

// the post-IDCT range-limit table of jdmaster.c indexed with (v & 1023)
__device__ __forceinline__ uint32_t idct_limit(int v) {
  const int x = v & 1023;
  return uint32_t(x < 128 ? x + 128 : (x < 512 ? 255 : (x < 896 ? 0 : x - 896)));
}

__global__ void __launch_bounds__(128) k_jpeg_idct(const JpegImg* __restrict__ imgs, const int16_t* __restrict__ coef, uint8_t* __restrict__ planes) {
  const JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  for (uint32_t blk = blockIdx.x * blockDim.x + threadIdx.x; blk < im.nblocks; blk += gridDim.x * blockDim.x) {
    const uint32_t m = blk / im.bpm;
    int b = int(blk - m * im.bpm);
    int c = 0;
    while (c + 1 < im.ncomp && b >= im.boff[c + 1]) ++c;
    b -= im.boff[c];
    const int my = int(m / im.mcux), mx = int(m - uint32_t(my) * im.mcux);
    const int by = my * im.vs[c] + b / im.hs[c], bx = mx * im.hs[c] + b % im.hs[c];
    const int4* src = reinterpret_cast<const int4*>(coef + (im.coef_off + blk) * 64);
    int d[64];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int4 v = src[i];
      const int16_t* h = reinterpret_cast<const int16_t*>(&v);
#pragma unroll
      for (int k = 0; k < 8; ++k) d[i * 8 + k] = int(h[k]) * int(im.q[c][i * 8 + k]);
    }
    int ws[64];
#pragma unroll
    for (int col = 0; col < 8; ++col) {
      int o[8];
      idct_1d(d[col], d[8 + col], d[16 + col], d[24 + col], d[32 + col], d[40 + col], d[48 + col], d[56 + col], o);
#pragma unroll
      for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (o[r] + (1 << 10)) >> 11;  // DESCALE(CONST_BITS - PASS1_BITS)
    }
    uint8_t* dst = planes + im.plane_off[c] + size_t(by * 8) * im.pw[c] + bx * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      int o[8];
      idct_1d(ws[r * 8], ws[r * 8 + 1], ws[r * 8 + 2], ws[r * 8 + 3], ws[r * 8 + 4], ws[r * 8 + 5], ws[r * 8 + 6], ws[r * 8 + 7], o);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        lo |= idct_limit((o[k] + (1 << 17)) >> 18) << (8 * k);  // DESCALE(CONST_BITS + PASS1_BITS + 3)
        hi |= idct_limit((o[k + 4] + (1 << 17)) >> 18) << (8 * k);
      }
      *reinterpret_cast<uint2*>(dst + size_t(r) * im.pw[c]) = make_uint2(lo, hi);
    }
  }
}

// one chroma sample of the upsampled plane at output (x, y) (libjpeg-turbo's fancy upsampling, jdsample.c; h2v1 / h2v2 planes
// at most 2 samples wide are replicated, as libjpeg-turbo then uses its plain upsampler)
__device__ __forceinline__ int chroma_at(const uint8_t* __restrict__ p, int pw, int cw, int ch, int fh, int fv, int x, int y) {
  if (fh == 1 && fv == 1) return p[size_t(y) * pw + x];
  const int xi = x >> (fh - 1), yi = y >> (fv - 1);
  if (fh == 2 && cw <= 2) return p[size_t(yi) * pw + xi];
  if (fv == 1) {  // h2v1
    const uint8_t* r = p + size_t(yi) * pw;
    return (x & 1) ? (3 * r[xi] + r[min(xi + 1, cw - 1)] + 2) >> 2 : (3 * r[xi] + r[max(xi - 1, 0)] + 1) >> 2;
  }
  const int yn = (y & 1) ? min(yi + 1, ch - 1) : max(yi - 1, 0);
  const uint8_t* r0 = p + size_t(yi) * pw;
  const uint8_t* r1 = p + size_t(yn) * pw;
  if (fh == 1) return (3 * r0[xi] + r1[xi] + ((y & 1) ? 2 : 1)) >> 2;  // h1v2
  const int xn = (x & 1) ? min(xi + 1, cw - 1) : max(xi - 1, 0);
  const int cs = 3 * r0[xi] + r1[xi], cn = 3 * r0[xn] + r1[xn];
  return (3 * cs + cn + ((x & 1) ? 7 : 8)) >> 4;
}

__device__ __forceinline__ uint8_t clamp_u8(int v) { return uint8_t(v < 0 ? 0 : (v > 255 ? 255 : v)); }

__global__ void __launch_bounds__(256) k_jpeg_color(const JpegImg* __restrict__ imgs, const uint8_t* __restrict__ planes) {
  const JpegImg& im = imgs[blockIdx.y];
  if (im.status) return;
  const int W = im.width, H = im.height;
  const uint8_t* py = planes + im.plane_off[0];
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < int64_t(W) * H; i += int64_t(gridDim.x) * blockDim.x) {
    const int y = int(i / W), x = int(i - int64_t(y) * W);
    const int Y = py[size_t(y) * im.pw[0] + x];
    uint8_t* o = im.out + size_t(y) * im.out_pitch + size_t(x) * 3;
    if (im.ncomp == 1) {
      o[0] = o[1] = o[2] = uint8_t(Y);
      continue;
    }
    const int cb = chroma_at(planes + im.plane_off[1], im.pw[1], im.cw[1], im.ch[1], im.hmax, im.vmax, x, y) - 128;
    const int cr = chroma_at(planes + im.plane_off[2], im.pw[2], im.cw[2], im.ch[2], im.hmax, im.vmax, x, y) - 128;
    // jdcolor.c build_ycc_rgb_table: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414) in 16-bit fixed point
    o[0] = clamp_u8(Y + ((91881 * cr + 32768) >> 16));
    o[1] = clamp_u8(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    o[2] = clamp_u8(Y + ((116130 * cb + 32768) >> 16));
  }
}

}  // namespace

struct JpegState {
  HostBuf stage;  // pinned: image table | Huffman tables | scan bytes
  DevBuf in, un, tiles, rst, exits, changed, bases, coef, planes;
  std::vector<JpegHuff> huff;
};

void jp_destroy(b2_context* ctx) {
  delete ctx->jp;
  ctx->jp = nullptr;
}

extern "C" int b2_jpeg_info_host(const uint8_t* data, size_t size, int* height, int* width, int* components) {
  HostHeader hd;
  const int rc = parse_header(data, size, hd);
  if (rc) return rc;
  if (height) *height = hd.height;
  if (width) *width = hd.width;
  if (components) *components = hd.ncomp;
  return 0;
}

extern "C" const char* b2_jpeg_status_string(int code) {
  switch (code) {
    case 0: return "ok";
    case J_LIMIT: return "beyond the size limits (16384 pixels a side, 2^26 pixels, 256 MiB a file)";
    case J_HEADER: return "not a JPEG file or a corrupt header";
    case J_PROGRESSIVE: return "progressive JPEG is not supported";
    case J_ARITH: return "arithmetic coding is not supported";
    case J_LOSSLESS: return "lossless / hierarchical JPEG is not supported";
    case J_PRECISION: return "only 8-bit samples are supported";
    case J_COMPONENTS: return "only 1 (gray) or 3 (YCbCr) components are supported (CMYK / YCCK are not)";
    case J_RGB: return "RGB colour space (Adobe transform 0) is not supported";
    case J_SAMPLING: return "sampling factors other than luma h1v1 / h2v1 / h1v2 / h2v2 with 1x1 chroma are not supported";
    case J_MULTISCAN: return "multi-scan JPEG (a scan without every component, or in another order) is not supported";
    case J_DNL: return "DNL (image height defined after the scan) is not supported";
    case J_TRUNCATED: return "truncated file (no EOI marker after the scan)";
    case J_CORRUPT: return "corrupt or truncated entropy-coded data";
    case J_HUFFTABLE: return "Huffman table with an all-ones code is not supported";
    default: return "unknown status";
  }
}

extern "C" int b2_jpeg_decode_batched_dev(b2_context* ctx, b2_jpeg_image* images, int n, void* stream) {
  if (!ctx || (!images && n > 0) || n < 0) return B2_ERR_ARG;
  if (n > JPEG_MAX_BATCH) return b2_fail(ctx, B2_ERR_ARG, "b2_jpeg_decode_batched_dev: more than 256 images");
  if (n == 0) return B2_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!ctx->jp) ctx->jp = new JpegState();
  JpegState& S = *ctx->jp;

  // host parse and layout
  std::vector<JpegImg> im(n);
  std::vector<int> idx;  // images that go to the device
  S.huff.clear();
  uint64_t in_bytes = 0, tiles = 0, subs = 0, segs = 0, blocks = 0, plane_bytes = 0;
  int max_tiles = 1, max_subs = 1, max_blocks = 1;
  int64_t max_pix = 1;
  for (int i = 0; i < n; ++i) {
    images[i].out_status = 0;
    images[i].out_rounds = 0;
    HostHeader hd;
    int rc = parse_header(images[i].data, images[i].size, hd);
    if (!rc && (!images[i].out || images[i].out_pitch < size_t(hd.width) * 3)) rc = J_LIMIT;
    if (rc) {
      images[i].out_status = rc;
      continue;
    }
    JpegImg& g = im[idx.size()];
    memset(&g, 0, sizeof(g));
    g.width = hd.width;
    g.height = hd.height;
    g.ncomp = hd.ncomp;
    g.hmax = hd.ncomp == 1 ? 1 : hd.c[0].h;
    g.vmax = hd.ncomp == 1 ? 1 : hd.c[0].v;
    g.mcux = cdiv(hd.width, 8 * g.hmax);
    g.mcuy = cdiv(hd.height, 8 * g.vmax);
    const int mcus = g.mcux * g.mcuy;
    g.ri = hd.restart ? hd.restart : mcus;
    g.nseg = uint32_t(cdiv(mcus, g.ri));
    g.bpm = 0;
    for (int c = 0; c < hd.ncomp; ++c) {
      g.hs[c] = hd.ncomp == 1 ? 1 : hd.c[c].h;
      g.vs[c] = hd.ncomp == 1 ? 1 : hd.c[c].v;
      g.boff[c] = g.bpm;
      g.bpm += g.hs[c] * g.vs[c];
      g.pw[c] = g.mcux * g.hs[c] * 8;
      g.ph[c] = g.mcuy * g.vs[c] * 8;
      g.cw[c] = cdiv(hd.width * g.hs[c], g.hmax);
      g.ch[c] = cdiv(hd.height * g.vs[c], g.vmax);
      g.plane_off[c] = plane_bytes;
      plane_bytes += (uint64_t(g.pw[c]) * g.ph[c] + 255) & ~uint64_t(255);
      const uint8_t* qt = hd.qt[hd.c[c].tq];
      for (int k = 0; k < 64; ++k) {
        static const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                       41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                       30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
        g.q[c][zz[k]] = hd.qprec[hd.c[c].tq] ? uint16_t((qt[2 * k] << 8) | qt[2 * k + 1]) : qt[k];
      }
    }
    g.nblocks = uint32_t(mcus) * g.bpm;
    g.coef_off = blocks;
    blocks += g.nblocks;
    g.huff = uint32_t(S.huff.size());
    S.huff.resize(S.huff.size() + 6);
    for (int c = 0; c < 3; ++c) {
      const int cc = c < hd.ncomp ? c : 0;
      build_huff(hd.ht[0][hd.c[cc].td], S.huff[g.huff + c]);
      build_huff(hd.ht[1][hd.c[cc].ta], S.huff[g.huff + 3 + c]);
    }
    g.in_len = uint32_t(images[i].size - hd.scan_off);
    g.in_off = in_bytes;
    in_bytes += (uint64_t(g.in_len) + JPEG_TILE - 1) / JPEG_TILE * JPEG_TILE + JPEG_TILE;
    g.tile0 = uint32_t(tiles);
    const int nt = cdiv(int(g.in_len), JPEG_TILE);
    tiles += nt;
    g.sub0 = uint32_t(subs);
    g.nsub_cap = uint32_t((uint64_t(g.in_len) * 8 + JPEG_SUB - 1) / JPEG_SUB + 1);
    subs += g.nsub_cap;
    g.rst0 = uint32_t(segs);
    segs += g.nseg;
    g.out = images[i].out;
    g.out_pitch = images[i].out_pitch;
    g.end = g.in_len;
    max_tiles = std::max(max_tiles, nt);
    max_subs = std::max(max_subs, int(g.nsub_cap));
    max_blocks = std::max(max_blocks, int(g.nblocks));
    max_pix = std::max(max_pix, int64_t(g.width) * g.height);
    idx.push_back(i);
  }
  const int m = int(idx.size());
  if (m == 0) return B2_OK;

  // one upload through pinned staging: image table | Huffman tables | scan bytes
  const size_t t_bytes = sizeof(JpegImg) * m, h_bytes = sizeof(JpegHuff) * S.huff.size();
  const size_t h_off = (t_bytes + 255) & ~size_t(255), b_off = (h_off + h_bytes + 255) & ~size_t(255);
  const size_t total = b_off + in_bytes;
  B2_CUDA(ctx, S.stage.ensure(total));
  uint8_t* hs = S.stage.as<uint8_t>();
  memcpy(hs, im.data(), t_bytes);
  memcpy(hs + h_off, S.huff.data(), h_bytes);
  for (int k = 0; k < m; ++k) memcpy(hs + b_off + im[k].in_off, images[idx[k]].data + (images[idx[k]].size - im[k].in_len), im[k].in_len);
  B2_CUDA(ctx, S.in.ensure(total));
  B2_CUDA(ctx, S.un.ensure(in_bytes));
  B2_CUDA(ctx, S.tiles.ensure(tiles * sizeof(uint64_t)));
  B2_CUDA(ctx, S.rst.ensure(std::max<uint64_t>(segs, 1) * sizeof(uint32_t)));
  B2_CUDA(ctx, S.exits.ensure(subs * sizeof(uint64_t)));
  B2_CUDA(ctx, S.bases.ensure(subs * sizeof(uint32_t)));
  B2_CUDA(ctx, S.changed.ensure(size_t(JPEG_ROUNDS + 1) * m * sizeof(int)));
  B2_CUDA(ctx, S.coef.ensure(blocks * 64 * sizeof(int16_t)));
  B2_CUDA(ctx, S.planes.ensure(plane_bytes));
  B2_CUDA(ctx, cudaMemcpyAsync(S.in.p, hs, total, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(S.changed.p, 0, size_t(JPEG_ROUNDS + 1) * m * sizeof(int), st));
  ctx->h2d_bytes += total;

  JpegImg* d_im = S.in.as<JpegImg>();
  const JpegHuff* d_huff = reinterpret_cast<const JpegHuff*>(S.in.as<uint8_t>() + h_off);
  const uint8_t* d_in = S.in.as<uint8_t>() + b_off;
  uint8_t* d_un = S.un.as<uint8_t>();
  uint64_t* d_tiles = S.tiles.as<uint64_t>();
  uint32_t* d_rst = S.rst.as<uint32_t>();
  uint64_t* d_ex = S.exits.as<uint64_t>();
  uint32_t* d_base = S.bases.as<uint32_t>();
  int* d_changed = S.changed.as<int>();
  int16_t* d_coef = S.coef.as<int16_t>();
  uint8_t* d_planes = S.planes.as<uint8_t>();
  const int gx_bytes = std::min(cdiv(max_tiles * JPEG_TILE, 256), 1024);
  B2_LAUNCH(ctx, k_jpeg_markers, dim3(gx_bytes, m), 256, 0, st, d_im, d_in);
  B2_LAUNCH(ctx, k_jpeg_count, dim3(std::min(max_tiles, 1024), m), 256, 0, st, d_im, d_in, d_tiles);
  B2_LAUNCH(ctx, k_jpeg_tiles, m, 1024, 0, st, d_im, d_tiles);
  B2_LAUNCH(ctx, k_jpeg_compact, dim3(std::min(max_tiles, 1024), m), 256, 0, st, d_im, d_in, d_tiles, d_un, d_rst);
  B2_CHECK_LAUNCH(ctx);
  const dim3 g_sub(std::min(cdiv(max_subs, 128), 4096), m);
  const int max_chunks = cdiv(max_subs, JPEG_CHUNK);
  B2_LAUNCH(ctx, k_jpeg_sync_chunk, dim3(std::min(max_chunks, 1024), m), JPEG_CHUNK, 0, st, d_im, d_un, d_rst, d_huff, d_ex);
  for (int r = 1; r <= JPEG_ROUNDS; ++r)
    B2_LAUNCH(ctx, k_jpeg_sync_round, dim3(cdiv(max_chunks, 128), m), 128, 0, st, d_im, d_un, d_rst, d_huff, d_ex, d_changed, r, m);
  B2_LAUNCH(ctx, k_jpeg_sync_serial, m, 32, 0, st, d_im, d_un, d_rst, d_huff, d_ex, d_changed, m);
  B2_LAUNCH(ctx, k_jpeg_bases, m, 1024, 0, st, d_im, d_ex, d_base);
  B2_LAUNCH(ctx, k_jpeg_write, g_sub, 128, 0, st, d_im, d_un, d_rst, d_huff, d_ex, d_base, d_coef);
  B2_CHECK_LAUNCH(ctx);
  B2_LAUNCH(ctx, k_jpeg_dc, dim3(3, m), 1024, 0, st, d_im, d_coef);
  B2_LAUNCH(ctx, k_jpeg_idct, dim3(std::min(cdiv(max_blocks, 128), 8192), m), 128, 0, st, d_im, d_coef, d_planes);
  B2_LAUNCH(ctx, k_jpeg_color, dim3(int(std::min<int64_t>((max_pix + 255) / 256, 8192)), m), 256, 0, st, d_im, d_planes);
  B2_CHECK_LAUNCH(ctx);
  B2_CUDA(ctx, cudaMemcpyAsync(hs, d_im, t_bytes, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  const JpegImg* res = reinterpret_cast<const JpegImg*>(hs);
  for (int k = 0; k < m; ++k) {
    images[idx[k]].out_status = res[k].status;
    images[idx[k]].out_rounds = res[k].rounds;
  }
  return B2_OK;
}
