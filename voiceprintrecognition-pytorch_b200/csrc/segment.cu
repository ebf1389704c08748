// Front of speaker diarization on the device (predict.py:365-379 with mvector/audio.py and
// infer_utils/speaker_diarization.py):
//   (a) frame energies of the energy VAD, the twin of
//         (x[:nf*hop].astype(float64).reshape(nf, hop) ** 2).mean(axis=1)
//       bit for bit.  numpy reduces each row with its pairwise sum: below 8 elements sequentially from 0.0; up to 128
//       with eight strided accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added in order;
//       above 128 split at n2 = n/2 - (n/2) % 8 and the two halves' sums added.  The squares of float32 values are
//       exact in float64, so __dadd_rn in that tree order and one __ddiv_rn by hop give numpy's result.  Eight lanes
//       work on one frame (lane j = accumulator j), so a warp holds four frames; the tree depends on hop alone, so
//       every lane of the grid walks the same tree and the shuffles stay warp-uniform.
//   (b) chunk windows: dst[i, j] = j < valid[i] ? src[offset[i] + j] : 0 for j < ld, one coalesced pass over dst.
// Every launch is asynchronous; no atomics: two calls give bit-identical results.
#include "kernels.cuh"

namespace vpb {

constexpr int FE_THREADS = 256;
constexpr int FE_GROUPS = FE_THREADS / 8;        // frames per CTA
constexpr int FE_DEPTH = 32;                     // split levels above the leaves: hop < 2^31 needs at most 25
constexpr int GW_THREADS = 256;
constexpr int GW_ITEMS = 4;                      // output samples per thread (strided by GW_THREADS: coalesced)

__device__ __forceinline__ int64_t pw_split(int64_t n) {
  const int64_t n2 = n / 2;
  return n2 - n2 % 8;
}

__device__ __forceinline__ double pw_sq(const float* a, int64_t i) {
  const double v = (double)__ldg(a + i);
  return __dmul_rn(v, v);
}

// One leaf of numpy's pairwise sum (n <= 128) over the squares of a[0 .. n): every lane of the 8-lane group returns it.
__device__ __forceinline__ double pw_leaf(const float* a, int64_t n, int j) {
  if (n < 8) {
    double r = 0.0;
    for (int64_t i = 0; i < n; ++i) r = __dadd_rn(r, pw_sq(a, i));
    return r;
  }
  const int64_t m = n - n % 8;
  double r = pw_sq(a, j);
  for (int64_t i = 8 + j; i < m; i += 8) r = __dadd_rn(r, pw_sq(a, i));
  // lanes j and j^1 (then ^2, ^4) hold the two operands of one node of ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)); the sum is
  // commutative, so both lanes form the same value
  r = __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 1));
  r = __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 2));
  r = __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 4));
  for (int64_t i = m; i < n; ++i) r = __dadd_rn(r, pw_sq(a, i));
  return r;
}

__global__ void __launch_bounds__(FE_THREADS) frame_energy_kernel(const float* __restrict__ x, int64_t nf, int64_t hop,
                                                                   double* __restrict__ out) {
  __shared__ double left[FE_GROUPS][FE_DEPTH];     // per frame: sums of the finished left children on the current path
  pdl_launch_dependents();
  pdl_wait();
  const int g = threadIdx.x >> 3, j = threadIdx.x & 7;
  const int64_t f = (int64_t)blockIdx.x * FE_GROUPS + g;
  const float* a = x + (f < nf ? f : nf - 1) * hop;   // frames past the end walk the tree too (uniform shuffles)
  // post-order walk of the split tree: (off, n) the current node, bit d of rbits set when the node at depth d + 1 of
  // the path is a right child
  int64_t off = 0, n = hop;
  int depth = 0;
  uint32_t rbits = 0;
  double s;
  for (;;) {
    while (n > 128) {
      n = pw_split(n);
      rbits &= ~(1u << depth);
      ++depth;
    }
    s = pw_leaf(a + off, n, j);
    while (depth > 0 && ((rbits >> (depth - 1)) & 1u)) {      // a right child: its parent is complete
      --depth;
      s = __dadd_rn(left[g][depth], s);
    }
    if (depth == 0) break;
    __syncwarp();                                               // the slot's previous readers are done
    if (j == 0) left[g][depth - 1] = s;
    __syncwarp();
    int64_t pn = hop, poff = 0;                                 // the parent node, from the root along rbits
    for (int d = 0; d < depth - 1; ++d) {
      const int64_t h = pw_split(pn);
      if ((rbits >> d) & 1u) { poff += h; pn -= h; } else { pn = h; }
    }
    const int64_t h = pw_split(pn);
    off = poff + h;
    n = pn - h;
    rbits |= 1u << (depth - 1);
  }
  if (j == 0 && f < nf) out[f] = __ddiv_rn(s, (double)hop);
}

__global__ void __launch_bounds__(GW_THREADS) gather_windows_kernel(const float* __restrict__ src,
                                                                     const int64_t* __restrict__ offset,
                                                                     const int32_t* __restrict__ valid, int64_t rows,
                                                                     int64_t ld, float* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t c0 = (int64_t)blockIdx.x * (GW_THREADS * GW_ITEMS) + threadIdx.x;
  for (int64_t r = blockIdx.y; r < rows; r += gridDim.y) {
    const int64_t v = valid[r];
    const float* s = src + offset[r];
    float* d = dst + r * ld;
#pragma unroll
    for (int k = 0; k < GW_ITEMS; ++k) {
      const int64_t c = c0 + k * GW_THREADS;
      if (c < ld) d[c] = c < v ? __ldg(s + c) : 0.f;
    }
  }
}

cudaError_t launch_frame_energy(const float* x, int64_t nf, int64_t hop, double* out, cudaStream_t stream) {
  const int64_t blocks = (nf + FE_GROUPS - 1) / FE_GROUPS;
  launch_pdl(frame_energy_kernel, dim3((unsigned)blocks), dim3(FE_THREADS), 0, stream, x, nf, hop, out);
  return cudaGetLastError();
}

cudaError_t launch_gather_windows(const float* src, const int64_t* offset, const int32_t* valid, int64_t rows, int64_t ld,
                                  float* dst, cudaStream_t stream) {
  const int64_t bx = (ld + GW_THREADS * GW_ITEMS - 1) / (GW_THREADS * GW_ITEMS);
  const unsigned by = (unsigned)(rows < 65535 ? rows : 65535);
  launch_pdl(gather_windows_kernel, dim3((unsigned)bx, by), dim3(GW_THREADS), 0, stream, src, offset, valid, rows, ld, dst);
  return cudaGetLastError();
}

}  // namespace vpb
