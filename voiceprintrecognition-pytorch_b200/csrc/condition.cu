// Input conditioning of the embedding path (predict.py:185-212, reader.py:82-107) on the device:
//   (a) polyphase resampler, the twin of scipy.signal.resample_poly(x.astype(float64), up, down) with the default
//       ('kaiser', 5.0) window and padtype='constant', rounded once to float32.  Ragged rows, each with its own
//       (up, down), in one launch.  Output j is upfirdn output i = j + n_pre_remove,
//         y[j] = sum_{k = kmin..kmax} (double)x[k] * hpad[i*down - k*up]
//       summed in increasing k from 0.0 with __dmul_rn / __dadd_rn (no contraction): scipy's own order, so the result
//       is bit-identical.  The taps hpad (n_pre_pad zeros + firwin * up) are stored per phase p = (i*down) % up,
//       tab[p * nt + m] = hpad[p + m*up], so a thread walks one contiguous row; each CTA stages its input window in
//       shared memory (global reads when the window does not fit: extreme down-sampling ratios only).
//   (b) dB gain, the twin of AudioSegment.normalize(target_db, max_gain_db): per-tile fp64 sums of the (exact) squares
//       combined in tile order, gain = target_db - 10 log10(sum / n), factor = 10^(gain / 20) in fp64, and every sample
//       x <- (float)(x * factor) -- the float64 product numpy forms for float32 samples times a float64 scalar.
//       gain > max_gain_db (including a silent row: +inf) sets the row's flag and leaves the row unscaled.
// Every launch is asynchronous; no atomics: two calls give bit-identical results.
#include "kernels.cuh"

namespace vpb {

constexpr int RS_THREADS = 256;                 // one output sample per thread
constexpr int RS_WINDOW = 4096;                 // staged input samples per CTA (16 KB)
constexpr int GN_THREADS = 256;
constexpr int GN_ITEMS = 16;
constexpr int GN_TILE = GN_THREADS * GN_ITEMS;  // samples per energy partial

struct RsFilter {
  int64_t Lh;            // padded filter length (n_pre_pad + 2 * half_len + 1)
  int64_t nt;            // taps per phase row
  int64_t n_pre_remove;
};

__host__ __device__ inline RsFilter rs_filter(int up, int down) {
  const int64_t max_rate = up > down ? up : down;
  const int64_t half_len = 10 * max_rate;
  const int64_t n_pre_pad = down - half_len % down;
  RsFilter f;
  f.Lh = n_pre_pad + 2 * half_len + 1;
  f.nt = (f.Lh + up - 1) / up;
  f.n_pre_remove = (half_len + n_pre_pad) / down;
  return f;
}

__device__ __forceinline__ int64_t rs_kmin(int64_t t0, int64_t Lh, int up) {
  const int64_t num = t0 - (Lh - 1);
  return num <= 0 ? 0 : (num + up - 1) / up;
}

__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const float* __restrict__ x, int64_t in_ld, float* __restrict__ y,
                                                               int64_t out_ld, const int64_t* __restrict__ n_in_v,
                                                               const int64_t* __restrict__ n_out_v, const int32_t* __restrict__ up_v,
                                                               const int32_t* __restrict__ down_v,
                                                               const int64_t* __restrict__ tap_off_v,
                                                               const double* __restrict__ taps) {
  __shared__ float win[RS_WINDOW];
  const int b = blockIdx.y;
  const int64_t j0 = (int64_t)blockIdx.x * RS_THREADS;
  const int64_t j = j0 + threadIdx.x;
  const int64_t n_in = n_in_v[b], n_out = n_out_v[b];
  const int up = up_v[b], down = down_v[b];
  const float* xr = x + (int64_t)b * in_ld;
  float* yr = y + (int64_t)b * out_ld;
  if (j0 >= n_out) {                              // padding only
    if (j < out_ld) yr[j] = 0.f;
    return;
  }
  if (up == down) {                               // rate already right: a copy
    if (j < out_ld) yr[j] = j < n_in ? xr[j] : 0.f;
    return;
  }
  const RsFilter f = rs_filter(up, down);
  const double* tab = taps + tap_off_v[b];
  // input window of the CTA's outputs j0 .. j_last (kmin / kmax grow with j)
  const int64_t j_last = min(j0 + RS_THREADS, n_out) - 1;
  const int64_t w_lo = rs_kmin((j0 + f.n_pre_remove) * down, f.Lh, up);
  const int64_t w_hi = min(n_in - 1, (j_last + f.n_pre_remove) * down / up);
  const bool staged = w_hi - w_lo + 1 <= RS_WINDOW;
  if (staged) {
    for (int64_t k = w_lo + threadIdx.x; k <= w_hi; k += RS_THREADS) win[k - w_lo] = xr[k];
    __syncthreads();
  }
  if (j >= out_ld) return;
  if (j >= n_out) {
    yr[j] = 0.f;
    return;
  }
  const int64_t t0 = (j + f.n_pre_remove) * down;
  const int64_t q = t0 / up;
  const int64_t p = t0 - q * up;
  const int64_t kmin = rs_kmin(t0, f.Lh, up);
  const int64_t kmax = min(n_in - 1, q);
  const double* row = tab + p * f.nt;             // row[q - k] = hpad[t0 - k*up]
  double acc = 0.0;
  if (staged) {
    for (int64_t k = kmin; k <= kmax; ++k) acc = __dadd_rn(acc, __dmul_rn((double)win[k - w_lo], __ldg(row + (q - k))));
  } else {
    for (int64_t k = kmin; k <= kmax; ++k) acc = __dadd_rn(acc, __dmul_rn((double)xr[k], __ldg(row + (q - k))));
  }
  yr[j] = (float)acc;
}

__global__ void __launch_bounds__(GN_THREADS) gain_energy_kernel(const float* __restrict__ w, int64_t ld,
                                                                  const int64_t* __restrict__ lens, int64_t ntiles,
                                                                  double* __restrict__ partial) {
  __shared__ double red[GN_THREADS];
  const int b = blockIdx.y;
  const int64_t n = lens[b];
  const int64_t base = (int64_t)blockIdx.x * GN_TILE;
  const float* xr = w + (int64_t)b * ld;
  double s = 0.0;
#pragma unroll 4
  for (int r = 0; r < GN_ITEMS; ++r) {
    const int64_t i = base + r * GN_THREADS + threadIdx.x;
    if (i < n) {
      const double v = (double)xr[i];
      s = __dadd_rn(s, __dmul_rn(v, v));
    }
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = GN_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[(int64_t)b * ntiles + blockIdx.x] = red[0];
}

__global__ void gain_factor_kernel(const int64_t* __restrict__ lens, int B, int64_t ntiles, const double* __restrict__ partial,
                                   double target_db, double max_gain_db, double* __restrict__ factor, int32_t* __restrict__ flags) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t n = lens[b];
  const int64_t used = (n + GN_TILE - 1) / GN_TILE;
  double s = 0.0;
  for (int64_t t = 0; t < used; ++t) s = __dadd_rn(s, partial[(int64_t)b * ntiles + t]);
  const double mean = __ddiv_rn(s, (double)n);
  const double gain = __dsub_rn(target_db, __dmul_rn(10.0, log10(mean)));
  const bool over = gain > max_gain_db;           // false for NaN: the row becomes NaN, as on the host
  flags[b] = over ? 1 : 0;
  factor[b] = over ? 1.0 : pow(10.0, __ddiv_rn(gain, 20.0));
}

__global__ void __launch_bounds__(GN_THREADS) gain_apply_kernel(float* __restrict__ w, int64_t ld, const int64_t* __restrict__ lens,
                                                                 const double* __restrict__ factor, const int32_t* __restrict__ flags) {
  const int b = blockIdx.y;
  if (flags[b]) return;
  const int64_t n = lens[b];
  const double fct = factor[b];
  float* xr = w + (int64_t)b * ld;
  const int64_t base = (int64_t)blockIdx.x * GN_TILE;
#pragma unroll 4
  for (int r = 0; r < GN_ITEMS; ++r) {
    const int64_t i = base + r * GN_THREADS + threadIdx.x;
    if (i < n) xr[i] = (float)__dmul_rn((double)xr[i], fct);
  }
}

cudaError_t launch_resample(const float* x, int64_t in_ld, float* y, int64_t out_ld, int B, const int64_t* n_in,
                            const int64_t* n_out, const int32_t* up, const int32_t* down, const int64_t* tap_off,
                            const double* taps, cudaStream_t stream) {
  const dim3 grid((unsigned)((out_ld + RS_THREADS - 1) / RS_THREADS), (unsigned)B);
  resample_kernel<<<grid, RS_THREADS, 0, stream>>>(x, in_ld, y, out_ld, n_in, n_out, up, down, tap_off, taps);
  return cudaGetLastError();
}

size_t gain_scratch_bytes(int B, int64_t ld) {
  const int64_t ntiles = (ld + GN_TILE - 1) / GN_TILE;
  return (size_t)B * (size_t)(ntiles + 1) * sizeof(double);
}

cudaError_t launch_gain(float* w, int64_t ld, int B, const int64_t* lens, double target_db, double max_gain_db,
                        int32_t* flags, void* scratch, cudaStream_t stream) {
  const int64_t ntiles = (ld + GN_TILE - 1) / GN_TILE;
  double* partial = (double*)scratch;
  double* factor = partial + (int64_t)B * ntiles;
  const dim3 grid((unsigned)ntiles, (unsigned)B);
  gain_energy_kernel<<<grid, GN_THREADS, 0, stream>>>(w, ld, lens, ntiles, partial);
  gain_factor_kernel<<<(B + 127) / 128, 128, 0, stream>>>(lens, B, ntiles, partial, target_db, max_gain_db, factor, flags);
  gain_apply_kernel<<<grid, GN_THREADS, 0, stream>>>(w, ld, lens, factor, flags);
  return cudaGetLastError();
}

}  // namespace vpb
