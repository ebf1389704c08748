// Uncompressed PCM container samples (WAV, RF64 / BW64, AIFF / AIFF-C) -> float32 mono rows on the device, the twin of
// mvector.pcm.to_mono bit for bit (include/vpb200.h states the conversion).  The host parses the headers
// (mvector/pcm.py); this pass only reads the sample bytes.
//
// A memory-bound elementwise pass: one thread converts PCM_ITEMS frames of a row, strided by the block so the float32
// stores of a warp are coalesced.  Samples start at any byte offset and can be 3 bytes wide, so every sample is read a
// byte at a time; neighbouring threads read neighbouring bytes, so each 32-byte sector still comes from DRAM once.  A
// row's info is checked before any of its bytes is read, and a refused row is written as zeros.
#include <algorithm>

#include "kernels.cuh"

namespace vpb {

constexpr int PCM_THREADS = 256;
constexpr int PCM_ITEMS = 4;                     // frames per thread, strided by PCM_THREADS

__device__ __forceinline__ int pcm_width(int fmt) {
  switch (fmt) {
    case VP_PCM_U8: case VP_PCM_S8: case VP_PCM_ULAW: case VP_PCM_ALAW: return 1;
    case VP_PCM_S16LE: case VP_PCM_S16BE: return 2;
    case VP_PCM_S24LE: case VP_PCM_S24BE: return 3;
    case VP_PCM_S32LE: case VP_PCM_S32BE: case VP_PCM_F32LE: case VP_PCM_F32BE: return 4;
    case VP_PCM_F64LE: case VP_PCM_F64BE: return 8;
    default: return 0;
  }
}

// ITU-T G.711 expansion to 16-bit linear.  mu-law: the complemented byte holds sign, 3-bit segment and 4-bit mantissa;
// |x| = (((mantissa << 3) + 0x84) << segment) - 0x84.  A-law: the byte XOR 0x55; |x| = (mantissa << 4) + 8 in segment 0,
// else ((mantissa << 4) + 0x108) << (segment - 1); a set sign bit is positive.
__device__ __forceinline__ int32_t ulaw_linear(uint32_t u) {
  u = ~u & 0xFFu;
  const int32_t t = ((((int32_t)(u & 0x0Fu) << 3) + 0x84) << ((u >> 4) & 7)) - 0x84;
  return (u & 0x80u) ? -t : t;
}

__device__ __forceinline__ int32_t alaw_linear(uint32_t a) {
  a ^= 0x55u;
  const int seg = (a >> 4) & 7;
  int32_t t = (int32_t)(a & 0x0Fu) << 4;
  t = seg == 0 ? t + 8 : (t + 0x108) << (seg - 1);
  return (a & 0x80u) ? t : -t;
}

// Unsigned little- / big-endian integer of n <= 8 bytes at p, any alignment.
__device__ __forceinline__ uint64_t load_le(const uint8_t* p, int n) {
  uint64_t v = 0;
  for (int k = n - 1; k >= 0; --k) v = (v << 8) | __ldg(p + k);
  return v;
}
__device__ __forceinline__ uint64_t load_be(const uint8_t* p, int n) {
  uint64_t v = 0;
  for (int k = 0; k < n; ++k) v = (v << 8) | __ldg(p + k);
  return v;
}

// One stored sample at p as float32: integers x / 2^(N-1), floats as stored (F64 rounded to nearest).
__device__ __forceinline__ float pcm_sample(const uint8_t* p, int fmt) {
  switch (fmt) {
    case VP_PCM_U8: return __fdiv_rn((float)((int32_t)__ldg(p) - 128), 128.f);
    case VP_PCM_S8: return __fdiv_rn((float)(int8_t)__ldg(p), 128.f);
    case VP_PCM_S16LE: return __fdiv_rn((float)(int16_t)load_le(p, 2), 32768.f);
    case VP_PCM_S16BE: return __fdiv_rn((float)(int16_t)load_be(p, 2), 32768.f);
    case VP_PCM_S24LE: return __fdiv_rn((float)((int32_t)((uint32_t)load_le(p, 3) << 8) >> 8), 8388608.f);
    case VP_PCM_S24BE: return __fdiv_rn((float)((int32_t)((uint32_t)load_be(p, 3) << 8) >> 8), 8388608.f);
    case VP_PCM_S32LE: return __fdiv_rn(__int2float_rn((int32_t)load_le(p, 4)), 2147483648.f);
    case VP_PCM_S32BE: return __fdiv_rn(__int2float_rn((int32_t)load_be(p, 4)), 2147483648.f);
    case VP_PCM_F32LE: return __uint_as_float((uint32_t)load_le(p, 4));
    case VP_PCM_F32BE: return __uint_as_float((uint32_t)load_be(p, 4));
    case VP_PCM_F64LE: return __double2float_rn(__longlong_as_double((long long)load_le(p, 8)));
    case VP_PCM_F64BE: return __double2float_rn(__longlong_as_double((long long)load_be(p, 8)));
    case VP_PCM_ULAW: return __fdiv_rn((float)ulaw_linear(__ldg(p)), 32768.f);
    default: return __fdiv_rn((float)alaw_linear(__ldg(p)), 32768.f);
  }
}

// numpy's float32 mean of a frame's ch = 1..8 samples (x.reshape(-1, ch).mean(axis=1)): the sum starts at +0.0 and runs
// left to right below 8 values, ((c0+c1)+(c2+c3))+((c4+c5)+(c6+c7)) for 8, then one division by ch.  One channel is
// the sample itself.  The same order as vp_flac_decode's warp shuffles (flac.cu), restated for one thread.
__device__ __forceinline__ float frame_mean(const uint8_t* p, int fmt, int w, int ch) {
  if (ch == 1) return pcm_sample(p, fmt);
  float acc;
  if (ch == 8) {
    const float s01 = __fadd_rn(pcm_sample(p, fmt), pcm_sample(p + w, fmt));
    const float s23 = __fadd_rn(pcm_sample(p + 2 * w, fmt), pcm_sample(p + 3 * w, fmt));
    const float s45 = __fadd_rn(pcm_sample(p + 4 * w, fmt), pcm_sample(p + 5 * w, fmt));
    const float s67 = __fadd_rn(pcm_sample(p + 6 * w, fmt), pcm_sample(p + 7 * w, fmt));
    acc = __fadd_rn(0.f, __fadd_rn(__fadd_rn(s01, s23), __fadd_rn(s45, s67)));
  } else {
    acc = 0.f;
    for (int c = 0; c < ch; ++c) acc = __fadd_rn(acc, pcm_sample(p + c * w, fmt));
  }
  return __fdiv_rn(acc, (float)ch);
}

// status of a row's info (include/vpb200.h): 0 or the OR of the reasons it is refused
__device__ __forceinline__ int32_t pcm_check(const vp_pcm_info& in, int64_t nbytes, int64_t ld) {
  int32_t st = 0;
  const int w = pcm_width(in.format);
  if (!w) st |= 1;
  if (in.channels < 1 || in.channels > 8) st |= 2;
  if (in.frames < 0 || in.frames > ld) st |= 4;
  const int64_t fb = (int64_t)(w ? w : 1) * min(max(in.channels, 1), 8);   // bytes per frame, 1..64
  if (in.byte_off < 0 || in.byte_off > nbytes || max(in.frames, (int64_t)0) > (nbytes - in.byte_off) / fb) st |= 8;
  return st;
}

__global__ void __launch_bounds__(PCM_THREADS) pcm_decode_kernel(const uint8_t* __restrict__ data, int64_t nbytes,
                                                                 const vp_pcm_info* __restrict__ info, int64_t ld,
                                                                 float* __restrict__ out, int32_t* __restrict__ status) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const vp_pcm_info in = info[b];
  const int32_t st = pcm_check(in, nbytes, ld);
  if (blockIdx.x == 0 && threadIdx.x == 0) status[b] = st;
  const int64_t n = st ? 0 : in.frames;
  const int fmt = in.format, ch = in.channels;
  const int w = pcm_width(fmt);
  const uint8_t* src = data + (st ? 0 : in.byte_off);
  float* row = out + (int64_t)b * ld;
  for (int64_t j0 = (int64_t)blockIdx.x * (PCM_THREADS * PCM_ITEMS); j0 < ld;
       j0 += (int64_t)gridDim.x * (PCM_THREADS * PCM_ITEMS)) {
#pragma unroll
    for (int k = 0; k < PCM_ITEMS; ++k) {
      const int64_t j = j0 + k * PCM_THREADS + threadIdx.x;
      if (j < ld) row[j] = j < n ? frame_mean(src + j * ch * w, fmt, w, ch) : 0.f;
    }
  }
}

cudaError_t launch_pcm_decode(const uint8_t* data, int64_t nbytes, const vp_pcm_info* info, int B, float* out,
                              int64_t ld, int32_t* status, cudaStream_t stream) {
  // a CTA per PCM_THREADS * PCM_ITEMS samples of each row, capped so a long row's CTAs loop instead
  const int64_t bx = std::max<int64_t>(1, std::min<int64_t>((ld + PCM_THREADS * PCM_ITEMS - 1) / (PCM_THREADS * PCM_ITEMS),
                                                            1 << 16));
  launch_pdl(pcm_decode_kernel, dim3((unsigned)bx, (unsigned)B), dim3(PCM_THREADS), 0, stream, data, nbytes, info, ld,
             out, status);
  return cudaGetLastError();
}

}  // namespace vpb
