// Batched FLAC decoder (RFC 9639) for 4-24 bits per sample: B native streams concatenated on the device -> B float32 mono
// rows at the native rate, each the twin of mvector.audio.pcm_to_mono on the decoded integers.
//
// Frames carry no length field and the sync code 0xFFF8 / 0xFFF9 may occur inside a payload, so the frames are found and
// proven in three passes before any sample is written:
//   scan   one thread per byte: a candidate is a sync code whose header parses (no reserved or invalid code) and passes
//          its CRC-8.
//   link   one thread per candidate: CRC-16 forward, stopping at the first later candidate (or the stream end) where the
//          two bytes before it equal the running CRC; the walk is bounded by STREAMINFO's maximum frame size (or, when
//          that is unset, by a verbatim-frame bound from the maximum block size).  A linked frame claims the slot
//          start / min_blocksize of the stream's frame table; two frames claiming one slot refuse the stream.
//   decode one warp per slot, lane c = channel c: each lane skips the subframes before its own (they are sequential in
//          the bitstream), then all lanes step through the block together, one sample per iteration, and lane 0 mixes
//          the channels (stereo decorrelation, float32 scaling, numpy's mean order) and writes the row.
// A stream is refused (status != 0, row contents unspecified) when its frames do not tile [0, total_samples) -- each
// frame's successor at its link end must start where it ends, the first frame sits at the first-frame offset, and the
// block sizes sum to total_samples -- when a frame contradicts STREAMINFO, when a subframe holds a reserved code or a
// value out of range, or when its decode does not end on the CRC-16 the link found.  Every read is bounded by the
// stream's own byte range and every write by total_samples <= ld.
#include <algorithm>

#include "kernels.cuh"

namespace vpb {

constexpr int FL_THREADS = 256;
constexpr int FL_DEC_THREADS = 128;                 // decode: one warp per frame slot
constexpr int FL_WARPS = FL_DEC_THREADS / 32;

enum : int32_t {
  FL_ERR_INFO = 1,        // STREAMINFO outside what the decoder takes, or the frame table would overflow max_frames
  FL_ERR_FIRST = 2,       // no proven frame at the first-frame offset
  FL_ERR_TILING = 4,      // frames overlap, leave a gap, or do not sum to total_samples
  FL_ERR_HEADER = 8,      // a frame header contradicts STREAMINFO
  FL_ERR_SUBFRAME = 16    // reserved code, out-of-range value, or the decode does not end at the frame's CRC-16
};

struct FlacHdr {
  int64_t start;          // first sample of the frame in the stream
  int32_t bs, rate, assign, nch, bps, len, variable;
};

__device__ __forceinline__ uint8_t crc8_byte(uint8_t c, uint8_t b) {
  c ^= b;
#pragma unroll
  for (int k = 0; k < 8; ++k) c = (uint8_t)((c & 0x80) ? (c << 1) ^ 0x07 : (c << 1));
  return c;
}

// Frame header at p (bytes before `end`): true when it parses without a reserved / invalid code and its CRC-8 matches.
__device__ bool parse_header(const uint8_t* __restrict__ d, int64_t p, int64_t end, const vp_flac_info& si, FlacHdr& h) {
  if (end - p < 6 || d[p] != 0xFF || (d[p + 1] & 0xFE) != 0xF8) return false;
  h.variable = d[p + 1] & 1;
  const int bsc = d[p + 2] >> 4, src = d[p + 2] & 15, chc = d[p + 3] >> 4, bpc = (d[p + 3] >> 1) & 7;
  if (bsc == 0 || src == 15 || chc > 10 || bpc == 3 || bpc == 7 || (d[p + 3] & 1)) return false;
  int64_t q = p + 4;
  const uint32_t c0 = d[q++];
  int extra;
  uint64_t num;
  if (c0 < 0x80) { extra = 0; num = c0; }
  else if (c0 >= 0xC0 && c0 < 0xE0) { extra = 1; num = c0 & 0x1F; }
  else if (c0 >= 0xE0 && c0 < 0xF0) { extra = 2; num = c0 & 0x0F; }
  else if (c0 >= 0xF0 && c0 < 0xF8) { extra = 3; num = c0 & 0x07; }
  else if (c0 >= 0xF8 && c0 < 0xFC) { extra = 4; num = c0 & 0x03; }
  else if (c0 >= 0xFC && c0 < 0xFE) { extra = 5; num = c0 & 0x01; }
  else if (c0 == 0xFE) { extra = 6; num = 0; }
  else return false;
  if (extra == 6 && !h.variable) return false;               // frame numbers have at most 31 bits
  if (end - q < extra + 3) return false;
  for (int k = 0; k < extra; ++k) {
    const uint32_t c = d[q++];
    if ((c & 0xC0) != 0x80) return false;
    num = (num << 6) | (c & 0x3F);
  }
  if (!h.variable && num >= (1ull << 31)) return false;
  if (bsc == 1) h.bs = 192;
  else if (bsc <= 5) h.bs = 576 << (bsc - 2);
  else if (bsc == 6) h.bs = 1 + d[q++];
  else if (bsc == 7) { h.bs = 1 + ((d[q] << 8) | d[q + 1]); q += 2; }
  else h.bs = 256 << (bsc - 8);
  if (end - q < 3) return false;
  switch (src) {
    case 0: h.rate = si.sample_rate; break;
    case 1: h.rate = 88200; break;
    case 2: h.rate = 176400; break;
    case 3: h.rate = 192000; break;
    case 4: h.rate = 8000; break;
    case 5: h.rate = 16000; break;
    case 6: h.rate = 22050; break;
    case 7: h.rate = 24000; break;
    case 8: h.rate = 32000; break;
    case 9: h.rate = 44100; break;
    case 10: h.rate = 48000; break;
    case 11: h.rate = 96000; break;
    case 12: h.rate = 1000 * d[q++]; break;
    default: h.rate = ((d[q] << 8) | d[q + 1]) * (src == 14 ? 10 : 1); q += 2;
  }
  h.bps = bpc == 0 ? si.bps : bpc == 1 ? 8 : bpc == 2 ? 12 : 12 + 4 * (bpc - 3);   // 4, 5, 6 -> 16, 20, 24
  h.assign = chc;
  h.nch = chc < 8 ? chc + 1 : 2;
  if (q >= end) return false;
  uint8_t c = 0;
  for (int64_t k = p; k < q; ++k) c = crc8_byte(c, d[k]);
  if (c != d[q]) return false;
  h.len = (int32_t)(q + 1 - p);
  h.start = h.variable ? (int64_t)num : (int64_t)num * si.max_blocksize;
  return true;
}

__device__ __forceinline__ int stream_of(const int64_t* __restrict__ off, int B, int64_t x) {
  int lo = 0, hi = B - 1;                          // last b with off[b] <= x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Frames a stream may hold: every frame but the last has at least min_blocksize samples.
__device__ __forceinline__ int64_t stream_slots(const vp_flac_info& si) {
  return (si.total_samples + si.min_blocksize - 1) / si.min_blocksize;
}

// Longest frame the link walk considers: STREAMINFO's maximum frame size, else a verbatim frame of the maximum block size.
__device__ __forceinline__ int64_t walk_bound(const vp_flac_info& si) {
  if (si.max_framesize > 0) return si.max_framesize;
  return 16 + (int64_t)si.channels * (6 + ((int64_t)si.max_blocksize * (si.bps + 1) + 7) / 8) + 2;
}

struct FlacScratch {
  uint8_t* cand;          // [nbytes] 1 = header candidate
  uint32_t* len;          // [nbytes] proven frame length at a candidate, else 0
  int64_t* slot;          // [max_frames] frame byte offset, -1 = empty
  int64_t* slot_base;     // [B + 1]
  unsigned long long* sum_bs;   // [B]
};

__global__ void flac_init_kernel(const int64_t* __restrict__ stream_off, const int64_t* __restrict__ frame_off,
                                 const vp_flac_info* __restrict__ info, int B, int64_t nbytes, int64_t ld,
                                 int64_t max_frames, FlacScratch s, int32_t* __restrict__ status) {
  // the stream ranges must be ordered and inside [0, nbytes): every later pass reads data and scratch by them
  __shared__ int bad_offsets;
  if (threadIdx.x == 0) bad_offsets = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    if (stream_off[b] < 0 || stream_off[b] > stream_off[b + 1] || stream_off[b + 1] > nbytes) bad_offsets = 1;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const vp_flac_info si = info[b];
    const bool ok = si.total_samples >= 1 && si.total_samples <= ld && si.channels >= 1 && si.channels <= 8 &&
                    si.bps >= 4 && si.bps <= 24 && si.min_blocksize >= 16 && si.max_blocksize >= si.min_blocksize &&
                    si.max_blocksize <= 65535 && si.max_framesize >= 0 && si.sample_rate > 0 &&
                    frame_off[b] >= stream_off[b] && frame_off[b] < stream_off[b + 1];
    status[b] = ok && !bad_offsets ? 0 : FL_ERR_INFO;
    s.sum_bs[b] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    for (int b = 0; b < B; ++b) {
      s.slot_base[b] = acc;
      if (status[b] == 0) acc += stream_slots(info[b]);
      if (acc > max_frames) { status[b] |= FL_ERR_INFO; acc = s.slot_base[b]; }
    }
    s.slot_base[B] = acc;
  }
}

__global__ void __launch_bounds__(FL_THREADS) flac_scan_kernel(const uint8_t* __restrict__ d, const int64_t* __restrict__ stream_off,
                                                               const int64_t* __restrict__ frame_off,
                                                               const vp_flac_info* __restrict__ info, int B, int64_t nbytes,
                                                               const int32_t* __restrict__ status, uint8_t* __restrict__ cand) {
  for (int64_t p = (int64_t)blockIdx.x * FL_THREADS + threadIdx.x; p < nbytes; p += (int64_t)gridDim.x * FL_THREADS) {
    uint8_t c = 0;
    if (d[p] == 0xFF) {
      const int b = stream_of(stream_off, B, p);
      FlacHdr h;                                   // parse_header reads nothing at or past the stream's end
      c = status[b] == 0 && p >= frame_off[b] && parse_header(d, p, stream_off[b + 1], info[b], h);
    }
    cand[p] = c;
  }
}

__global__ void __launch_bounds__(FL_THREADS) flac_link_kernel(const uint8_t* __restrict__ d, const int64_t* __restrict__ stream_off,
                                                               const vp_flac_info* __restrict__ info, int B, int64_t nbytes,
                                                               FlacScratch s, int32_t* __restrict__ status) {
  __shared__ uint16_t tab[256];
  for (int i = threadIdx.x; i < 256; i += FL_THREADS) {
    uint16_t c = (uint16_t)(i << 8);
    for (int k = 0; k < 8; ++k) c = (uint16_t)((c & 0x8000) ? (c << 1) ^ 0x8005 : (c << 1));
    tab[i] = c;
  }
  __syncthreads();
  for (int64_t p = (int64_t)blockIdx.x * FL_THREADS + threadIdx.x; p < nbytes; p += (int64_t)gridDim.x * FL_THREADS) {
    uint32_t L = 0;
    if (s.cand[p]) {
      const int b = stream_of(stream_off, B, p);
      const vp_flac_info si = info[b];
      FlacHdr h;
      parse_header(d, p, stream_off[b + 1], si, h);
      const int64_t lim = min(stream_off[b + 1], p + walk_bound(si));
      // crc = CRC-16 of [p, q - 2): a frame [p, q) ends with the big-endian CRC-16 of everything before it
      uint16_t crc = 0;
      int64_t q = p + h.len + 3;
      for (int64_t k = p; k < q - 2; ++k) crc = (uint16_t)((crc << 8) ^ tab[(crc >> 8) ^ d[k]]);
      for (; q <= lim; ++q) {
        if ((q == stream_off[b + 1] || s.cand[q]) && crc == (uint16_t)((d[q - 2] << 8) | d[q - 1])) {
          L = (uint32_t)(q - p);
          break;
        }
        crc = (uint16_t)((crc << 8) ^ tab[(crc >> 8) ^ d[q - 2]]);
      }
      if (L) {
        const int64_t slot = h.start / si.min_blocksize;
        if (h.start < 0 || slot >= stream_slots(si)) {
          atomicOr(status + b, FL_ERR_TILING);
        } else if (atomicCAS((unsigned long long*)(s.slot + s.slot_base[b] + slot), ~0ull, (unsigned long long)p) != ~0ull) {
          atomicOr(status + b, FL_ERR_TILING);
        }
      }
    }
    s.len[p] = L;
  }
}

// Bit reader over bytes [pos, end) of one frame: a 64-bit window, MSB first.  Reading past `end` sets `bad` and yields 0.
struct BitReader {
  const uint8_t* d;
  int64_t pos, end;
  uint64_t cache;
  int n;
  bool bad;

  __device__ void init(const uint8_t* data, int64_t bitpos, int64_t end_) {
    d = data; pos = bitpos >> 3; end = end_; cache = 0; n = 0; bad = false;
    read((int)(bitpos & 7));
  }
  __device__ __forceinline__ void refill() {
    while (n <= 56 && pos < end) { cache |= (uint64_t)d[pos++] << (56 - n); n += 8; }
  }
  __device__ __forceinline__ int64_t bitpos() const { return pos * 8 - n; }
  __device__ __forceinline__ uint32_t read(int k) {          // 0 <= k <= 32
    if (k == 0) return 0;
    if (n < k) refill();
    if (n < k) { bad = true; return 0; }
    const uint32_t v = (uint32_t)(cache >> (64 - k));
    cache <<= k;
    n -= k;
    return v;
  }
  __device__ __forceinline__ int32_t read_signed(int k) {    // k-bit two's complement, 0 <= k <= 32
    if (k == 0) return 0;
    const uint32_t v = read(k);
    return k == 32 ? (int32_t)v : (int32_t)(v << (32 - k)) >> (32 - k);
  }
  // zeros before the next 1 bit (consumed too); more than `limit` zeros sets `bad`
  __device__ __forceinline__ uint32_t unary(uint32_t limit) {
    uint32_t z = 0;
    while (true) {
      if (n == 0) refill();
      if (n == 0) { bad = true; return 0; }
      const int lz = cache ? __clzll((long long)cache) : 64;
      if (lz >= n) {
        z += n; cache = 0; n = 0;
      } else {
        z += lz; cache <<= lz + 1; n -= lz + 1;
        return z;
      }
      if (z > limit) { bad = true; return 0; }
    }
  }
};

// One subframe, decoded a sample at a time.
struct Subframe {
  int type;               // 0 CONSTANT, 1 VERBATIM, 2 FIXED / LPC
  int order, shift, sbits, wasted, bs;
  int32_t cval;
  int32_t coef[32];       // coef[j] multiplies the sample j + 1 steps back
  int32_t hist[32];       // hist[31] = the previous sample
  bool lpc, res_started, first_part;
  int pbits, esc, rk, psize;
  int32_t parts_left, in_part;

  __device__ void begin(BitReader& r, int bits, int bs_) {
    bs = bs_;
    if (r.read(1)) r.bad = true;                             // zero padding bit
    const int t = (int)r.read(6);
    wasted = 0;
    if (r.read(1)) wasted = (int)r.unary(32) + 1;
    sbits = bits - wasted;
    if (sbits < 1) r.bad = true;
    res_started = false;
    order = 0; shift = 0; lpc = false;
    if (t == 0) { type = 0; cval = r.read_signed(sbits); }
    else if (t == 1) type = 1;
    else if (t >= 8 && t <= 12) { type = 2; order = t - 8; }
    else if (t >= 32) { type = 2; order = t - 31; lpc = true; }
    else { r.bad = true; type = 0; cval = 0; }
    if (order > bs) r.bad = true;
#pragma unroll
    for (int j = 0; j < 32; ++j) { hist[j] = 0; coef[j] = 0; }
  }

  __device__ void start_residual(BitReader& r) {
    res_started = true;
    if (lpc) {
      const int prec = (int)r.read(4) + 1;
      if (prec == 16) r.bad = true;
      shift = r.read_signed(5);
      if (shift < 0) r.bad = true;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < order) coef[j] = r.read_signed(prec);
    } else {
      // fixed predictors as integer LPC coefficients (shift 0): exact
      coef[0] = order;
      coef[1] = order == 2 ? -1 : order == 3 ? -3 : order == 4 ? -6 : 0;
      coef[2] = order == 3 ? 1 : order == 4 ? 4 : 0;
      coef[3] = order == 4 ? -1 : 0;
    }
    const uint32_t method = r.read(2);
    if (method > 1) r.bad = true;
    pbits = method ? 5 : 4;
    const int po = (int)r.read(4);
    psize = bs >> po;
    if ((psize << po) != bs || psize < order) r.bad = true;
    parts_left = 1 << po;
    in_part = 0;
    first_part = true;
  }

  __device__ __forceinline__ void next_partition(BitReader& r) {
    const int param = (int)r.read(pbits);
    if (param == (1 << pbits) - 1) { esc = (int)r.read(5); } else { esc = -1; rk = param; }
    in_part = first_part ? psize - order : psize;
    first_part = false;
    --parts_left;
  }

  __device__ __forceinline__ int32_t residual(BitReader& r) {
    while (in_part == 0) {
      if (parts_left == 0 || r.bad) { r.bad = true; return 0; }
      next_partition(r);
    }
    --in_part;
    if (esc >= 0) return r.read_signed(esc);
    const uint32_t q = r.unary(0xFFFFFFFFu >> rk);
    if (q > (0xFFFFFFFFu >> rk)) { r.bad = true; return 0; }
    const uint32_t u = (q << rk) | r.read(rk);
    return (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
  }

  __device__ __forceinline__ void push(int32_t v) {
#pragma unroll
    for (int j = 0; j < 31; ++j) hist[j] = hist[j + 1];
    hist[31] = v;
  }

  // sample i (before the wasted-bits shift)
  __device__ __forceinline__ int32_t next(BitReader& r, int i) {
    if (type == 0) return cval;
    if (type == 1 || i < order) {
      const int32_t v = r.read_signed(sbits);
      if (type == 2) push(v);
      return v;
    }
    if (!res_started) start_residual(r);
    const int32_t e = residual(r);
    long long acc = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < order) acc += (long long)coef[j] * hist[31 - j];
    const long long v = (acc >> shift) + e;
    const long long lim = 1ll << (sbits - 1);
    if (v < -lim || v >= lim) r.bad = true;
    push((int32_t)v);
    return (int32_t)v;
  }

  __device__ void finish(BitReader& r) {
    if (type != 2) return;
    if (!res_started) start_residual(r);
    if (parts_left > 0 && first_part && psize == order) next_partition(r);   // a first partition with no samples
    if (parts_left != 0 || in_part != 0) r.bad = true;
  }
};

__device__ __forceinline__ int sub_bits(int assign, int bps, int c) {
  const bool side = (assign == 8 && c == 1) || (assign == 9 && c == 0) || (assign == 10 && c == 1);
  return bps + (side ? 1 : 0);
}

__global__ void __launch_bounds__(FL_DEC_THREADS, 1) flac_decode_kernel(const uint8_t* __restrict__ d,
                                                                 const int64_t* __restrict__ stream_off,
                                                                 const int64_t* __restrict__ frame_off,
                                                                 const vp_flac_info* __restrict__ info, int B,
                                                                 FlacScratch s, float* __restrict__ out, int64_t ld,
                                                                 int32_t* __restrict__ status) {
  const int64_t w = (int64_t)blockIdx.x * FL_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= s.slot_base[B]) return;
  const int64_t p = s.slot[w];
  if (p < 0) return;
  const int b = stream_of(s.slot_base, B, w);
  const vp_flac_info si = info[b];
  const int64_t send = stream_off[b + 1];
  FlacHdr h;
  parse_header(d, p, send, si, h);                         // proven by the scan
  const int64_t fend = p + s.len[p];
  int32_t err = 0;
  if (h.rate != si.sample_rate || h.bps != si.bps || h.nch != si.channels || h.bs > si.max_blocksize)
    err |= FL_ERR_HEADER;
  if (h.start + h.bs > si.total_samples) err |= FL_ERR_TILING;
  else if (h.bs < si.min_blocksize && h.start + h.bs != si.total_samples) err |= FL_ERR_HEADER;
  if ((p == frame_off[b]) != (h.start == 0)) err |= FL_ERR_TILING;
  if (fend < send) {                                       // the successor must be a proven frame starting where this ends
    FlacHdr n;
    if (!s.len[fend] || !parse_header(d, fend, send, si, n) || n.start != h.start + h.bs || n.variable != h.variable)
      err |= FL_ERR_TILING;
  } else if (h.start + h.bs != si.total_samples) {
    err |= FL_ERR_TILING;
  }
  if (err) {
    if (lane == 0) atomicOr(status + b, err);
    return;
  }
  if (lane == 0) atomicAdd(s.sum_bs + b, (unsigned long long)h.bs);

  const int nch = h.nch;
  const bool active = lane < nch;
  BitReader r;
  r.init(d, (p + h.len) * 8, fend - 2);
  Subframe sf;
  for (int c = 0; active && c < lane; ++c) {              // skip the subframes before this lane's own
    sf.begin(r, sub_bits(h.assign, h.bps, c), h.bs);
    for (int i = 0; i < h.bs && !r.bad; ++i) sf.next(r, i);
    sf.finish(r);
  }
  if (active) sf.begin(r, sub_bits(h.assign, h.bps, lane), h.bs);
  const float scale = (float)(1 << (h.bps - 1));
  float* row = out + (int64_t)b * ld + h.start;
  for (int i = 0; i < h.bs; ++i) {
    int32_t x = 0;
    if (active) x = sf.next(r, i) << sf.wasted;
    float y;
    if (h.assign >= 8) {
      const int32_t a = __shfl_sync(0xFFFFFFFFu, x, 0), c = __shfl_sync(0xFFFFFFFFu, x, 1);
      int32_t lft, rgt;
      if (h.assign == 8) { lft = a; rgt = a - c; }
      else if (h.assign == 9) { lft = a + c; rgt = c; }
      else { const int32_t m = (int32_t)(((uint32_t)a << 1) | (uint32_t)(c & 1)); lft = (m + c) >> 1; rgt = (m - c) >> 1; }
      const int32_t lim = 1 << (h.bps - 1);
      if (lft < -lim || lft >= lim || rgt < -lim || rgt >= lim) r.bad = true;
      y = __fdiv_rn(__fadd_rn(__fdiv_rn((float)lft, scale), __fdiv_rn((float)rgt, scale)), 2.f);
    } else {
      const float f = __fdiv_rn((float)x, scale);
      if (nch == 8) {                                      // numpy: ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7))
        const float s1 = __fadd_rn(f, __shfl_down_sync(0xFFFFFFFFu, f, 1));
        const float s2 = __fadd_rn(s1, __shfl_down_sync(0xFFFFFFFFu, s1, 2));
        const float s4 = __fadd_rn(s2, __shfl_down_sync(0xFFFFFFFFu, s2, 4));
        y = __fdiv_rn(s4, 8.f);
      } else {                                             // numpy: left to right below 8 values
        float acc = f;
        for (int c = 1; c < nch; ++c) acc = __fadd_rn(acc, __shfl_sync(0xFFFFFFFFu, f, c));
        y = nch == 1 ? f : __fdiv_rn(acc, (float)nch);
      }
    }
    if (lane == 0) row[i] = y;
  }
  if (active) {
    sf.finish(r);
    if (lane == nch - 1) {                                 // the last subframe ends, zero padded, at the CRC-16
      const int64_t bp = r.bitpos();
      const int pad = (int)((8 - (bp & 7)) & 7);
      if (r.read(pad) != 0 || r.bitpos() != (fend - 2) * 8) r.bad = true;
    }
    if (r.bad) atomicOr(status + b, FL_ERR_SUBFRAME);
  }
}

__global__ void flac_finish_kernel(const int64_t* __restrict__ frame_off, const vp_flac_info* __restrict__ info, int B,
                                   FlacScratch s, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || status[b]) return;
  if (!s.len[frame_off[b]]) status[b] |= FL_ERR_FIRST;
  else if ((int64_t)s.sum_bs[b] != info[b].total_samples) status[b] |= FL_ERR_TILING;
}

__global__ void __launch_bounds__(FL_THREADS) flac_pad_kernel(const vp_flac_info* __restrict__ info, float* __restrict__ out,
                                                              int64_t ld) {
  const int b = blockIdx.y;
  const int64_t n = max((int64_t)0, min(info[b].total_samples, ld));
  for (int64_t j = n + (int64_t)blockIdx.x * FL_THREADS + threadIdx.x; j < ld; j += (int64_t)gridDim.x * FL_THREADS)
    out[(int64_t)b * ld + j] = 0.f;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t flac_scratch_bytes(int B, int64_t nbytes, int64_t max_frames) {
  return align256((size_t)nbytes) + align256((size_t)nbytes * 4) + align256((size_t)max_frames * 8) +
         align256((size_t)(B + 1) * 8) + align256((size_t)B * 8);
}

cudaError_t launch_flac_decode(const uint8_t* data, int64_t nbytes, const int64_t* stream_off, const int64_t* frame_off,
                               const vp_flac_info* info, int B, int64_t max_frames, float* out, int64_t ld,
                               int32_t* status, void* scratch, cudaStream_t stream) {
  uint8_t* base = (uint8_t*)scratch;
  FlacScratch s;
  s.cand = base; base += align256((size_t)nbytes);
  s.len = (uint32_t*)base; base += align256((size_t)nbytes * 4);
  s.slot = (int64_t*)base; base += align256((size_t)max_frames * 8);
  s.slot_base = (int64_t*)base; base += align256((size_t)(B + 1) * 8);
  s.sum_bs = (unsigned long long*)base;
  cudaError_t e;
  if (max_frames > 0 && (e = cudaMemsetAsync(s.slot, 0xFF, (size_t)max_frames * 8, stream)) != cudaSuccess) return e;
  flac_init_kernel<<<1, 256, 0, stream>>>(stream_off, frame_off, info, B, nbytes, ld, max_frames, s, status);
  const unsigned gb = (unsigned)std::min<int64_t>((nbytes + FL_THREADS - 1) / FL_THREADS, 1 << 20);
  if (nbytes > 0) {
    flac_scan_kernel<<<gb, FL_THREADS, 0, stream>>>(data, stream_off, frame_off, info, B, nbytes, status, s.cand);
    flac_link_kernel<<<gb, FL_THREADS, 0, stream>>>(data, stream_off, info, B, nbytes, s, status);
  }
  if (max_frames > 0)
    flac_decode_kernel<<<(unsigned)((max_frames + FL_WARPS - 1) / FL_WARPS), FL_DEC_THREADS, 0, stream>>>(
        data, stream_off, frame_off, info, B, s, out, ld, status);
  flac_finish_kernel<<<(B + 127) / 128, 128, 0, stream>>>(frame_off, info, B, s, status);
  const dim3 pg((unsigned)std::max<int64_t>(1, std::min<int64_t>((ld + FL_THREADS - 1) / FL_THREADS, 4096)), (unsigned)B);
  flac_pad_kernel<<<pg, FL_THREADS, 0, stream>>>(info, out, ld);
  return cudaGetLastError();
}

}  // namespace vpb
