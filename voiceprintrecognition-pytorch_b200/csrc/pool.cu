// Whole-utterance reductions and elementwise glue of the backbones (all channel-last, lane <-> channel so every
// warp-level load is a coalesced 128 B row segment):
//   colstats   : SE squeeze (ecapa_tdnn.py:79, resnet_se.py:58-60), ASP global mean/std (pooling.py:91-94,108),
//                CAM++ StatsPool (campplus.py:27-33), TSTP (pooling.py:140-148), CAM++ context (campplus.py:96-111)
//   asp_pool   : softmax over time + attentive mean/std (pooling.py:120-126)
//   ew         : SE excite + residual (ecapa_tdnn.py:84,143; resnet_se.py:40-44), AFF blend (eres2net.py:48-50)
#include "kernels.cuh"

namespace vpb {

// Per-channel sum (or max) over the 8 warps of a 256-thread CTA with lane = channel; every thread gets its channel's
// total.  Fixed order (warp 0, 1, ..., 7), so results are deterministic.  Ends on a barrier: the caller may reduce again
// right away.
__device__ __forceinline__ float block_reduce(float v, bool is_max) {
  __shared__ float red[8][33];
  __shared__ float bc[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  red[wid][lane] = v;
  __syncthreads();
  if (wid == 0) {
    float s = red[0][lane];
#pragma unroll
    for (int i = 1; i < 8; ++i) s = is_max ? fmaxf(s, red[i][lane]) : s + red[i][lane];
    bc[lane] = s;
  }
  __syncthreads();
  const float r = bc[lane];
  __syncthreads();
  return r;
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src, bool valid) {
  const unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int bytes = valid ? 16 : 0;                       // src-size 0: the 16 destination bytes are zero filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(gmem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Stage rows [0, R) of a [.., ld] matrix, 32 columns starting at column c0 (only columns < C are read; C % 4 == 0), into
// dst[r * 32 + col]: 8 lanes x 16 B cover one 128-byte row, and every request of the CTA is in flight at once (one trip
// to HBM instead of rounds of register-staged loads).
__device__ __forceinline__ void stage_strip(float* dst, const float* src, int ld, int R, int c0, int C) {
  const int c4 = (threadIdx.x & 7) * 4;
  const bool cok = c0 + c4 < C;
  const float* g = src + c0 + c4;
  for (int r = threadIdx.x >> 3; r < R; r += blockDim.x >> 3)
    cp_async16(dst + r * 32 + c4, cok ? g + (size_t)r * ld : src, cok);
}

// Second statistic of the non-segment colstats modes from the centred sum of squares.
__device__ __forceinline__ float colstats_spread(const StatsParams& p, float ssq) {
  if (p.mode == VP_STATS_MEAN_STD_CLAMP) return sqrtf(fmaxf(ssq / (float)p.R, p.eps));
  if (p.mode == VP_STATS_MEAN_VAR_UNBIASED) return ssq / (float)(p.R - 1);
  if (p.mode == VP_STATS_MEAN_STD_UNBIASED) return sqrtf(ssq / (float)(p.R - 1));
  return sqrtf(ssq / (float)(p.R - 1) + p.eps);
}

// grid (ceil(C/32), B), block 256 = 8 warps; lane = channel, warps stride over the R rows.
__global__ void __launch_bounds__(256) colstats_kernel(const __grid_constant__ StatsParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const int b = blockIdx.y;
  const bool ok = c < p.C;
  const float* x = p.src + (size_t)b * p.R * p.in_ld + p.in_coff + c;

  if (p.mode == VP_STATS_SEG_CONTEXT) {
    // context[b, s, c] = mean_T(x) + mean over segment s (last segment divides by its in-bounds length)
    __shared__ float segsum[64][32];
    if (p.n_seg > 64) {
      // very long audio (> 64 segments = 128 s at CAM++'s 100-frame segments after the stride-2 TDNN): two sweeps -- the
      // utterance total first, then one segment at a time -- instead of parking the segment sums in shared memory
      float v = 0.f;
      if (ok) for (int r = wid; r < p.R; r += 8) v += x[(size_t)r * p.in_ld];
      const float mean = block_reduce(v, false) / (float)p.R;
      for (int s = 0; s < p.n_seg; ++s) {
        const int r0 = s * p.seg_len, r1 = min(r0 + p.seg_len, p.R);
        float u = 0.f;
        if (ok) for (int r = r0 + wid; r < r1; r += 8) u += x[(size_t)r * p.in_ld];
        const float ss = block_reduce(u, false);
        if (wid == 0 && ok) p.dst[((size_t)b * p.n_seg + s) * p.out_ld + p.out_coff + c] = mean + ss / (float)(r1 - r0);
      }
      return;
    }
    float total = 0.f;
    for (int s = 0; s < p.n_seg; ++s) {
      const int r0 = s * p.seg_len, r1 = min(r0 + p.seg_len, p.R);
      float v = 0.f;
      if (ok) for (int r = r0 + wid; r < r1; r += 8) v += x[(size_t)r * p.in_ld];
      const float ss = block_reduce(v, false);
      if (wid == 0) segsum[s][lane] = ss;
      total += ss;
    }
    if (wid == 0 && ok) {
      const float mean = total / (float)p.R;
      for (int s = 0; s < p.n_seg; ++s) {
        const int cnt = min(p.seg_len, p.R - s * p.seg_len);
        p.dst[((size_t)b * p.n_seg + s) * p.out_ld + p.out_coff + c] = mean + segsum[s][lane] / (float)cnt;
      }
    }
    return;
  }

  float v = 0.f;
  if (ok) for (int r = wid; r < p.R; r += 8) v += x[(size_t)r * p.in_ld];
  const float mean = block_reduce(v, false) / (float)p.R;
  float* o = p.dst + (size_t)b * p.out_ld + p.out_coff;
  if (p.mode == VP_STATS_MEAN) {
    if (wid == 0 && ok) o[c] = mean;
    return;
  }
  float q = 0.f;
  if (ok) for (int r = wid; r < p.R; r += 8) { float d = x[(size_t)r * p.in_ld] - mean; q = fmaf(d, d, q); }
  const float ssq = block_reduce(q, false);
  if (wid == 0 && ok) {
    o[c] = mean;
    o[p.C + c] = colstats_spread(p, ssq);
  }
}

// The non-segment modes with the whole [R, 32] strip staged in shared memory (1-D maps): one trip to HBM, then the
// same two-pass mean / centred sum of squares as colstats_kernel, out of shared memory.
__global__ void __launch_bounds__(256) colstats_smem_kernel(const __grid_constant__ StatsParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  extern __shared__ __align__(16) float sm[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32;
  const int c = c0 + lane;
  const int b = blockIdx.y;
  const bool ok = c < p.C;
  stage_strip(sm, p.src + (size_t)b * p.R * p.in_ld + p.in_coff, p.in_ld, p.R, c0, p.C);
  cp_async_wait_all();
  __syncthreads();
  float v = 0.f;
  for (int r = wid; r < p.R; r += 8) v += sm[r * 32 + lane];
  const float mean = block_reduce(v, false) / (float)p.R;
  float* o = p.dst + (size_t)b * p.out_ld + p.out_coff;
  if (p.mode == VP_STATS_MEAN) {
    if (wid == 0 && ok) o[c] = mean;
    return;
  }
  float q = 0.f;
  for (int r = wid; r < p.R; r += 8) { float d = sm[r * 32 + lane] - mean; q = fmaf(d, d, q); }
  const float ssq = block_reduce(q, false);
  if (wid == 0 && ok) {
    o[c] = mean;
    o[p.C + c] = colstats_spread(p, ssq);
  }
}

cudaError_t launch_colstats(const StatsParams& p, cudaStream_t stream) {
  dim3 grid((p.C + 31) / 32, p.B);
  const size_t smem = (size_t)p.R * 32 * sizeof(float);
  // up to 100 KB of strip, so that two CTAs per SM keep loads and sweeps overlapped
  if (p.mode != VP_STATS_SEG_CONTEXT && smem <= 100 * 1024 && (p.C & 3) == 0 && (p.in_ld & 3) == 0 && (p.in_coff & 3) == 0) {
    static PerDeviceSmem once;
    if (once.need(smem)) {
      cudaError_t e = cudaFuncSetAttribute(colstats_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
      if (e != cudaSuccess) return e;
      once.set(100 * 1024);
    }
    launch_pdl(colstats_smem_kernel, grid, 256, smem, stream, p);
    return cudaGetLastError();
  }
  launch_pdl(colstats_kernel, grid, 256, 0, stream, p);
  return cudaGetLastError();
}

// Attentive statistics: alpha = softmax_t(logit[b, t, c]); mean = sum alpha x; std = sqrt(clamp(sum alpha (x-mean)^2, eps)).
// x: src (in_ld/in_coff), logits: src2 (l_ld/l_coff); dst[b, c] = mean, dst[b, C + c] = std.
// Reads x and logits from global memory in three sweeps (L2-resident): for T > 800 and unaligned views.
__global__ void __launch_bounds__(256) asp_pool_kernel(const __grid_constant__ AspParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const int b = blockIdx.y;
  const bool ok = c < p.C;
  const float* x = p.x + (size_t)b * p.T * p.x_ld + p.x_coff + c;
  const float* l = p.logit + (size_t)b * p.T * p.l_ld + p.l_coff + c;

  float mx = -INFINITY;
  if (ok) for (int t = wid; t < p.T; t += 8) mx = fmaxf(mx, l[(size_t)t * p.l_ld]);
  mx = block_reduce(mx, true);
  float se = 0.f, sx = 0.f;
  if (ok) for (int t = wid; t < p.T; t += 8) {
    const float e = expf(l[(size_t)t * p.l_ld] - mx);
    se += e;
    sx = fmaf(e, x[(size_t)t * p.x_ld], sx);
  }
  se = block_reduce(se, false);
  sx = block_reduce(sx, false);
  const float mean = sx / se;
  float sq = 0.f;
  if (ok) for (int t = wid; t < p.T; t += 8) {
    const float e = expf(l[(size_t)t * p.l_ld] - mx);
    const float d = x[(size_t)t * p.x_ld] - mean;
    sq = fmaf(e, d * d, sq);
  }
  sq = block_reduce(sq, false);
  if (wid == 0 && ok) {
    float* o = p.dst + (size_t)b * p.out_ld + p.out_coff;
    o[c] = mean;
    if (!p.mean_only) o[p.C + c] = sqrtf(fmaxf(sq / se, p.eps));
  }
}

// Same computation with the [T, 32-column] strips of x and logits staged once in shared memory (each read from HBM
// once, coalesced 128 B rows), then the three softmax / mean / variance sweeps run out of shared memory.
__global__ void __launch_bounds__(256) asp_pool_smem_kernel(const __grid_constant__ AspParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  extern __shared__ __align__(16) float sm[];
  float* sx = sm;                       // [T][32]
  float* sl = sm + (size_t)p.T * 32;    // [T][32]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32;
  const int c = c0 + lane;
  const int b = blockIdx.y;
  const bool ok = c < p.C;
  stage_strip(sx, p.x + (size_t)b * p.T * p.x_ld + p.x_coff, p.x_ld, p.T, c0, p.C);
  stage_strip(sl, p.logit + (size_t)b * p.T * p.l_ld + p.l_coff, p.l_ld, p.T, c0, p.C);
  cp_async_wait_all();
  __syncthreads();
  float mx = -INFINITY;
  for (int t = wid; t < p.T; t += 8) mx = fmaxf(mx, sl[t * 32 + lane]);
  mx = block_reduce(mx, true);
  float se = 0.f, sxe = 0.f;
  for (int t = wid; t < p.T; t += 8) {
    const float e = expf(sl[t * 32 + lane] - mx);
    sl[t * 32 + lane] = e;                              // keep exp() for the variance sweep
    se += e;
    sxe = fmaf(e, sx[t * 32 + lane], sxe);
  }
  se = block_reduce(se, false);
  sxe = block_reduce(sxe, false);
  const float mean = sxe / se;
  float sq = 0.f;
  for (int t = wid; t < p.T; t += 8) {
    const float d = sx[t * 32 + lane] - mean;
    sq = fmaf(sl[t * 32 + lane], d * d, sq);
  }
  sq = block_reduce(sq, false);
  if (wid == 0 && ok) {
    float* o = p.dst + (size_t)b * p.out_ld + p.out_coff;
    o[c] = mean;
    if (!p.mean_only) o[p.C + c] = sqrtf(fmaxf(sq / se, p.eps));
  }
}

cudaError_t launch_asp_pool(const AspParams& p, cudaStream_t stream) {
  dim3 grid((p.C + 31) / 32, p.B);
  const size_t smem = (size_t)p.T * 32 * 2 * sizeof(float);
  if (smem <= 200 * 1024 && (p.C & 3) == 0 && (p.x_ld & 3) == 0 && (p.x_coff & 3) == 0 && (p.l_ld & 3) == 0 && (p.l_coff & 3) == 0) {
    static PerDeviceSmem once;
    if (once.need(smem)) {
      cudaError_t e = cudaFuncSetAttribute(asp_pool_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e != cudaSuccess) return e;
      once.set(200 * 1024);
    }
    launch_pdl(asp_pool_smem_kernel, grid, 256, smem, stream, p);
    return cudaGetLastError();
  }
  launch_pdl(asp_pool_kernel, grid, 256, 0, stream, p);
  return cudaGetLastError();
}

// Elementwise ops over [rows, C] (C % 4 == 0), float4 vectorised.
__global__ void __launch_bounds__(256) ew_kernel(const __grid_constant__ EwParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int c4n = p.C >> 2;
  const long long total = p.rows * c4n;
  float tmax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / c4n;
    const int c = (int)(i - m * c4n) * 4;
    float4 v = *reinterpret_cast<const float4*>(p.x + m * p.x_ld + p.x_coff + c);
    if (p.mode == VP_EW_GATE_RES) {
      if (p.gate) {
        const long long b = m / p.rows_per_utt;
        const float4 g = *reinterpret_cast<const float4*>(p.gate + b * p.C + c);
        v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
      }
      if (p.res) {
        const float4 r = *reinterpret_cast<const float4*>(p.res + m * p.res_ld + p.res_coff + c);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      v.x = apply_act(v.x, p.act2); v.y = apply_act(v.y, p.act2); v.z = apply_act(v.z, p.act2); v.w = apply_act(v.w, p.act2);
    } else if (p.mode == VP_EW_AFF) {
      const float4 y = *reinterpret_cast<const float4*>(p.y + m * p.y_ld + p.y_coff + c);
      const float4 a = *reinterpret_cast<const float4*>(p.att + m * p.att_ld + p.att_coff + c);
      float ax = 1.f + tanhf(a.x), ay = 1.f + tanhf(a.y), az = 1.f + tanhf(a.z), aw = 1.f + tanhf(a.w);
      v.x = v.x * ax + y.x * (2.f - ax);
      v.y = v.y * ay + y.y * (2.f - ay);
      v.z = v.z * az + y.z * (2.f - az);
      v.w = v.w * aw + y.w * (2.f - aw);
    }
    *reinterpret_cast<float4*>(p.dst + m * p.out_ld + p.out_coff + c) = v;
    tmax = amax4(tmax, v);
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

// dst[r, 0:C_out] = (x[r, 0:C], 0 ...): scalar, for feature dims that are not multiples of 4 (Spectrogram's n_fft/2+1 bins)
__global__ void __launch_bounds__(256) pad_copy_kernel(const __grid_constant__ EwParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const long long total = p.rows * p.C_out;
  float tmax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / p.C_out;
    const int c = (int)(i - m * p.C_out);
    const float v = c < p.C ? __ldg(p.x + m * p.x_ld + p.x_coff + c) : 0.f;
    p.dst[m * p.out_ld + p.out_coff + c] = v;
    tmax = fmaxf(tmax, fabsf(v));
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

cudaError_t launch_ew(const EwParams& p, cudaStream_t stream) {
  if (p.mode == VP_EW_PAD_COPY) {
    long long blocks = (p.rows * p.C_out + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    launch_pdl(pad_copy_kernel, (int)(blocks < 1 ? 1 : blocks), 256, 0, stream, p);
    return cudaGetLastError();
  }
  long long total = p.rows * (p.C >> 2);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (blocks < 1) blocks = 1;
  launch_pdl(ew_kernel, (int)blocks, 256, 0, stream, p);
  return cudaGetLastError();
}

// KTxKF pooling on a channel-last [B, T, F, C] map (column window in/out), float4 over channels.
//   mode 0: nn.MaxPool2d(k, stride, padding)                      (res2net.py:105)
//   mode 1: nn.AvgPool2d(k, stride, padding), count_include_pad   (res2net.py:33-34: divide by KT*KF always)
__global__ void __launch_bounds__(256) pool2d_kernel(const __grid_constant__ PoolParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int c4n = p.C >> 2;
  const long long total = (long long)p.B * p.Tout * p.Fout * c4n;
  float tmax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4n) * 4;
    long long m = i / c4n;
    const int fo = (int)(m % p.Fout);
    m /= p.Fout;
    const int to = (int)(m % p.Tout);
    const int b = (int)(m / p.Tout);
    float4 acc = p.mode == 0 ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int kt = 0; kt < p.KT; ++kt) {
      const int ti = to * p.sT - p.padT + kt;
      if (ti < 0 || ti >= p.Tin) continue;
      for (int kf = 0; kf < p.KF; ++kf) {
        const int fi = fo * p.sF - p.padF + kf;
        if (fi < 0 || fi >= p.Fin) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(p.src + ((size_t)(b * p.Tin + ti) * p.Fin + fi) * p.in_ld + p.in_coff + c));
        if (p.mode == 0) { acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w); }
        else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
      }
    }
    if (p.mode == 1) {
      const float inv = 1.f / (float)(p.KT * p.KF);
      acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    }
    *reinterpret_cast<float4*>(p.dst + ((size_t)(b * p.Tout + to) * p.Fout + fo) * p.out_ld + p.out_coff + c) = acc;
    tmax = amax4(tmax, acc);
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

cudaError_t launch_pool2d(const PoolParams& p, cudaStream_t stream) {
  long long total = (long long)p.B * p.Tout * p.Fout * (p.C >> 2);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (blocks < 1) blocks = 1;
  launch_pdl(pool2d_kernel, (int)blocks, 256, 0, stream, p);
  return cudaGetLastError();
}

}  // namespace vpb

// ---------------------------------------------------------------------------------------------------------------
// Cosine score matrix  out[i, j] = <a_i, b_j> / (|a_i| |b_j|)  for a [n, D], b [m, D] (row-major, any D >= 1):
// the scoring half of the callers around the embedding path -- voiceprint retrieval against the enrolled means
// (predict.py:169-183), trial-vs-enrol scoring of evaluate (trainer.py:454-461, sklearn cosine_similarity) and the
// similarity matrix of the diarization clustering (speaker_diarization.py:254-257).  One CTA = 32 x 32 scores, the two
// row blocks staged through shared memory in K chunks of 64, norms accumulated from the same tiles; fixed summation
// order -> deterministic, and a score does not depend on where its pair sits in the matrix.
// A zero-norm row scores 0 against everything, as sklearn's normalize() leaves a zero row zero: its norm is taken as 1,
// and its dot products are +0.  The CTAs of one grid row walk the tile rows with a stride of gridDim.y, which is capped
// at 65535, so every n and m up to INT32_MAX launches.
// ---------------------------------------------------------------------------------------------------------------
namespace vpb {

constexpr int COS_GRID_Y_MAX = 65535;

__global__ void __launch_bounds__(256) cosine_scores_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                                            int n, int m, int D, int a_ld, int b_ld, int out_ld) {
  __shared__ float sa[32][65], sb[32][65];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // thread -> column j = tx, rows ty, ty+8, ty+16, ty+24
  const int j0 = blockIdx.x * 32;
  for (long long i0 = (long long)blockIdx.y * 32; i0 < n; i0 += (long long)gridDim.y * 32) {
    float dot[4] = {0.f, 0.f, 0.f, 0.f}, na[4] = {0.f, 0.f, 0.f, 0.f}, nb = 0.f;
    for (int k0 = 0; k0 < D; k0 += 64) {
      for (int e = threadIdx.x; e < 32 * 64; e += 256) {
        const int r = e >> 6, c = e & 63;
        sa[r][c] = (i0 + r < n && k0 + c < D) ? __ldg(a + (size_t)(i0 + r) * a_ld + k0 + c) : 0.f;
        sb[r][c] = (j0 + r < m && k0 + c < D) ? __ldg(b + (size_t)(j0 + r) * b_ld + k0 + c) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int c = 0; c < 64; ++c) {
        const float bv = sb[tx][c];
        nb = fmaf(bv, bv, nb);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float av = sa[ty + 8 * q][c];
          dot[q] = fmaf(av, bv, dot[q]);
          na[q] = fmaf(av, av, na[q]);
        }
      }
      __syncthreads();
    }
    const int j = j0 + tx;
    const float rb = nb == 0.f ? 1.f : sqrtf(nb);
    if (j < m)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const long long i = i0 + ty + 8 * q;
        if (i < n) out[(size_t)i * out_ld + j] = dot[q] / ((na[q] == 0.f ? 1.f : sqrtf(na[q])) * rb);
      }
  }
}

cudaError_t launch_cosine_scores(const float* a, const float* b, float* out, int n, int m, int D, cudaStream_t stream) {
  const long long tiles_n = (n + 31LL) / 32;
  dim3 grid((unsigned)((m + 31LL) / 32), (unsigned)(tiles_n < COS_GRID_Y_MAX ? tiles_n : COS_GRID_Y_MAX));
  cosine_scores_kernel<<<grid, 256, 0, stream>>>(a, b, out, n, m, D, D, D, m);
  return cudaGetLastError();
}

}  // namespace vpb
