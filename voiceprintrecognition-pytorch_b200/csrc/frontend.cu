// Fused front-end: framing -> (DC removal, pre-emphasis) -> window -> real FFT -> power -> sparse mel -> log,
// one kernel, waveform read once from HBM through a shared-memory stage; then CMN + length mask.
//
// Replaces the reference's per-utterance Python loop over torchaudio.compliance.kaldi.fbank
// (mvector/data_utils/featurizer.py:119-132 -> kaldi.py:514-645: ~250 ATen ops per utterance, window and mel bank
// rebuilt on every call) and torchaudio.transforms.MelSpectrogram (featurizer.py:41-42,76), followed by
// AudioFeaturizer.forward's transpose / mean-subtract / mask (featurizer.py:77-90).
//
// The same kernel serves torchaudio.transforms.Spectrogram (identity "mel" bank, featurizer.py:43-44) and the mel stage
// of torchaudio.transforms.MFCC (featurizer.py:45-46), whose AmplitudeToDB / top_db clamp / DCT-II run in mfcc_post_kernel.
//
// FFT: two real frames are packed into one complex length-N Stockham autosort FFT held in shared memory.
// N = 2^a 3^b 5^c (4 | N): radix-8 passes first, then radix 4 / 2, then generic radix-5 / radix-3 passes (torchaudio's
// default n_fft = 400 = 8*2*5*5); the pass plan comes from the host.  A group of G threads (a multiple of 32, G ~ N/8)
// owns one FFT and synchronises on its own named barrier, 256/G groups per CTA run independently.
//
// PRECISION.  The window pipeline runs in fp32 op for op like the reference (those roundings are part of what the
// reference computes); the FFT, the power spectrum and the mel accumulation run in FP64 and are rounded to fp32 once.
// Why: the log turns the RELATIVE error of a mel energy into an absolute error, and with pre-emphasised input the
// low-frequency bins sit 30 dB below the frame's energy, so an fp32 FFT's absolute rounding error (any fp32 FFT, the
// reference's included) is ~1e-4 relative THERE.  Measured (tools/fbank_precision_study.py, 16 x 3 s of the bench input):
// torchaudio's own fp32 result is up to 6.1e-4 (log units) away from the exact value of its own formula, an fp32
// Stockham up to 4.1e-4, this kernel <= 2e-6.  The distance to the reference is therefore the REFERENCE's rounding
// error; no fp32 implementation can be closer to it than that without replicating its FFT library bit for bit.
// Cost: the FFT is shared-memory bound, radix 8 in fp64 moves the same bytes as radix 4 in fp32 did.
// Bound: the algorithmic traffic is 4*L + 4*T*F bytes per utterance (HBM); the kernel is shared-memory bound (DESIGN.md).
#include "kernels.cuh"

namespace vpb {

// ---- complex double helpers (the FFT runs in fp64: see the header comment) ----
struct cd { double x, y; };
__device__ __forceinline__ cd cadd(cd a, cd b) { return {a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ cd csub(cd a, cd b) { return {a.x - b.x, a.y - b.y}; }
__device__ __forceinline__ cd cmul(cd a, cd b) { return {a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
__device__ __forceinline__ cd cmi(cd a) { return {a.y, -a.x}; }                       // a * (-i)
__device__ __forceinline__ cd ld2(const double2* p) { const double2 v = *p; return {v.x, v.y}; }
__device__ __forceinline__ void st2(double2* p, cd v) { *p = make_double2(v.x, v.y); }

// barrier over the G threads of one FFT group (G % 32 == 0; ids 1..8, id 0 is __syncthreads)
__device__ __forceinline__ void group_sync(int g, int G) { asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "r"(G) : "memory"); }

__global__ void __launch_bounds__(256) frontend_kernel(const __grid_constant__ FrontendParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = p.N, WL = p.WL, F = p.F;
  const int G = p.G;                                // threads per FFT (multiple of 32)
  const int NG = 256 / G;                           // concurrent FFTs per CTA
  const int span = (p.fpb - 1) * p.hop + WL;

  double2* tw = reinterpret_cast<double2*>(smem_raw);               // N
  double2* bufA = tw + N;                                           // NG * N
  double2* bufB = bufA + (size_t)NG * N;                            // NG * N
  float* stage = reinterpret_cast<float*>(bufB + (size_t)NG * N);   // span floats (rounded up to x4)
  float* win = stage + ((span + 3) & ~3);                           // WL
  float* means = win + ((WL + 3) & ~3);                             // NG * 2
  float* red = means + NG * 2;                                      // 8 floats: per-warp maxima (MFCC mel stage)

  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * p.fpb;
  const int g = tid / G;
  const int t = tid - g * G;
  float vmax = -INFINITY;
  const float* wv = p.wave + (size_t)b * p.L;

  // ---- stage the waveform span, window and twiddles; the frame mode maps each staged sample to its source ----
  const int q0 = f0 * p.hop;
  for (int i = tid; i < span; i += 256) {
    int s = q0 + i;
    if (p.kind == 1) {                      // torch.stft of x zero-extended by p.pad at both ends: functional.py:112-134
      const int Lp = p.L + 2 * p.pad;
      if (p.frame != VP_FRAME_STFT_NOCENTER) s -= N / 2;
      if (p.frame == VP_FRAME_DEFAULT) {                  // reflect
        if (s < 0) s = -s;
        if (s >= Lp) s = 2 * (Lp - 1) - s;
      } else if (p.frame == VP_FRAME_STFT_REPLICATE) {
        s = min(max(s, 0), Lp - 1);
      } else if (p.frame == VP_FRAME_STFT_CIRCULAR) {
        if (s < 0) s += Lp;
        if (s >= Lp) s -= Lp;
      }                                                   // constant / not centred: outside is zero
      s -= p.pad;
    } else if (p.frame == VP_FRAME_KALDI_REFLECT) {       // kaldi._get_strided(snip_edges=False): x[-1-j] / x[2L-1-j]
      s -= p.pad;
      if (s < 0) s = -1 - s;
      if (s >= p.L) s = 2 * p.L - 1 - s;
    }
    stage[i] = (s >= 0 && s < p.L) ? __ldg(wv + s) : 0.f;
  }
  for (int i = tid; i < WL; i += 256) win[i] = __ldg(p.window + i);
  for (int i = tid; i < N; i += 256) tw[i] = __ldg(p.twiddle + i);
  __syncthreads();

  // Every group owns the frame pairs g, g + NG, ... of the CTA's tile and runs them start to finish on its own named
  // barrier: the groups never wait for each other inside the loop.
  const int npairs = p.fpb / 2;
  double2* src0 = bufA + (size_t)g * N;
  double2* dst0 = bufB + (size_t)g * N;
  for (int pair = g; pair < npairs; pair += NG) {
    const int fa = f0 + pair * 2;                   // frames packed as real (fa) and imaginary (fa + 1) parts
    const int oa = (fa - f0) * p.hop;
    const bool va = fa < p.T, vb = fa + 1 < p.T;
    if (!va) break;                                 // uniform over the group: frames beyond T (last tile of the utterance)

    // ---- per-frame mean (kaldi.py:183-186), one warp per frame ----
    float ma = 0.f, mb = 0.f;
    if (p.kind == 0 && p.remove_dc) {
      const int w = t >> 5, lane = t & 31;
      if (G >= 64) {
        if (w < 2) {
          const int o = oa + w * p.hop;
          float s = 0.f;
          if (w == 0 || vb)
            for (int j = lane; j < WL; j += 32) s += stage[o + j];
          s = warp_sum(s);
          if (lane == 0) means[g * 2 + w] = s / (float)WL;
        }
      } else {                                      // one warp per group: both frames, one after the other
        for (int w2 = 0; w2 < 2; ++w2) {
          const int o = oa + w2 * p.hop;
          float s = 0.f;
          if (w2 == 0 || vb)
            for (int j = lane; j < WL; j += 32) s += stage[o + j];
          s = warp_sum(s);
          if (lane == 0) means[g * 2 + w2] = s / (float)WL;
        }
      }
      group_sync(g, G);
      ma = means[g * 2];
      mb = means[g * 2 + 1];
    }
    // ---- window pipeline in fp32, op for op as kaldi.py:183-204 / torch.stft's window multiply; FFT input in fp64 ----
    for (int j = t; j < N; j += G) {
      float ya = 0.f, yb = 0.f;
      if (j < WL) {
        const int jp = j > 0 ? j - 1 : 0;
        const float wj = win[j];
        {
          float x = stage[oa + j];
          if (p.kind == 0) {
            x = __fsub_rn(x, ma);
            if (p.preemph != 0.f) x = __fsub_rn(x, __fmul_rn(p.preemph, __fsub_rn(stage[oa + jp], ma)));
          }
          ya = __fmul_rn(x, wj);
        }
        if (vb) {
          float x = stage[oa + p.hop + j];
          if (p.kind == 0) {
            x = __fsub_rn(x, mb);
            if (p.preemph != 0.f) x = __fsub_rn(x, __fmul_rn(p.preemph, __fsub_rn(stage[oa + p.hop + jp], mb)));
          }
          yb = __fmul_rn(x, wj);
        }
      }
      src0[j] = make_double2((double)ya, (double)yb);
    }
    group_sync(g, G);

    // ---- Stockham autosort FFT in fp64, pass plan from the host (radix 8 / 4 / 2, then 5 / 3) ----
    double2* src = src0;
    double2* dst = dst0;
    int Ns = 1;
    for (int ps = 0; ps < p.n_pass; ++ps) {
      const int R = p.radix[ps];
      const int q = N / R;
      const int step = q / Ns;                      // N / (Ns * R)
      const bool pow2 = (Ns & (Ns - 1)) == 0;
      for (int j = t; j < q; j += G) {
        const int kk = pow2 ? (j & (Ns - 1)) : (j % Ns);
        const int base = (j - kk) * R + kk;
        if (R == 8) {
          cd v[8];
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            v[r] = ld2(src + j + r * q);
            if (r > 0 && Ns > 1) v[r] = cmul(v[r], ld2(tw + r * kk * step));
          }
          const cd a0 = cadd(v[0], v[4]), a1 = csub(v[0], v[4]), a2 = cadd(v[2], v[6]), a3 = cmi(csub(v[2], v[6]));
          const cd a4 = cadd(v[1], v[5]), a5 = csub(v[1], v[5]), a6 = cadd(v[3], v[7]), a7 = cmi(csub(v[3], v[7]));
          const cd b0 = cadd(a0, a2), b2 = csub(a0, a2), b1 = cadd(a1, a3), b3 = csub(a1, a3);
          const cd b4 = cadd(a4, a6), b6 = cmi(csub(a4, a6));
          const double h = 0.70710678118654752440;
          const cd s5 = cadd(a5, a7), d5 = csub(a5, a7);
          const cd b5 = {h * (s5.x + s5.y), h * (s5.y - s5.x)};          // * (1 - i) / sqrt 2
          const cd b7 = {h * (d5.y - d5.x), -h * (d5.x + d5.y)};         // * (-1 - i) / sqrt 2
          st2(dst + base, cadd(b0, b4));          st2(dst + base + Ns, cadd(b1, b5));
          st2(dst + base + 2 * Ns, cadd(b2, b6)); st2(dst + base + 3 * Ns, cadd(b3, b7));
          st2(dst + base + 4 * Ns, csub(b0, b4)); st2(dst + base + 5 * Ns, csub(b1, b5));
          st2(dst + base + 6 * Ns, csub(b2, b6)); st2(dst + base + 7 * Ns, csub(b3, b7));
        } else if (R == 4) {
          cd v0 = ld2(src + j), v1 = ld2(src + j + q), v2 = ld2(src + j + 2 * q), v3 = ld2(src + j + 3 * q);
          if (Ns > 1) {
            v1 = cmul(v1, ld2(tw + kk * step));
            v2 = cmul(v2, ld2(tw + 2 * kk * step));
            v3 = cmul(v3, ld2(tw + 3 * kk * step));
          }
          const cd a0 = cadd(v0, v2), a1 = csub(v0, v2), a2 = cadd(v1, v3), a3 = cmi(csub(v1, v3));
          st2(dst + base, cadd(a0, a2));          st2(dst + base + Ns, cadd(a1, a3));
          st2(dst + base + 2 * Ns, csub(a0, a2)); st2(dst + base + 3 * Ns, csub(a1, a3));
        } else if (R == 2) {
          const cd v0 = ld2(src + j);
          cd v1 = ld2(src + j + q);
          if (Ns > 1) v1 = cmul(v1, ld2(tw + kk * step));
          st2(dst + base, cadd(v0, v1));
          st2(dst + base + Ns, csub(v0, v1));
        } else {
          // generic odd radix (5 or 3): out[m] = sum_r v[r] * W_R^(r m), W_R^k = tw[k * N / R]
          cd v[5];
#pragma unroll
          for (int r = 0; r < 5; ++r)
            if (r < R) {
              v[r] = ld2(src + j + r * q);
              if (r > 0 && Ns > 1) v[r] = cmul(v[r], ld2(tw + r * kk * step));
            }
#pragma unroll
          for (int m = 0; m < 5; ++m)
            if (m < R) {
              cd acc = v[0];
#pragma unroll
              for (int r = 1; r < 5; ++r)
                if (r < R) acc = cadd(acc, cmul(v[r], ld2(tw + ((r * m) % R) * q)));
              st2(dst + base + m * Ns, acc);
            }
        }
      }
      group_sync(g, G);
      double2* tmp = src; src = dst; dst = tmp;
      Ns *= R;
    }

    // ---- split the packed spectrum, power in fp64 (kaldi.py:616-618) into P[2][N/2+1] (reuses the idle FFT buffer) ----
    const int NB = N / 2 + 1;
    double* P = reinterpret_cast<double*>(dst);
    for (int k = t; k < NB; k += G) {
      const cd z = ld2(src + k);
      const cd zn = ld2(src + (k == 0 ? 0 : N - k));
      const double ar = 0.5 * (z.x + zn.x), ai = 0.5 * (z.y - zn.y);
      const double br = 0.5 * (z.y + zn.y), bi = -0.5 * (z.x - zn.x);
      double pa = ar * ar + ai * ai, pb = br * br + bi * bi;
      if (p.power == 1) { pa = sqrt(pa); pb = sqrt(pb); }
      if (p.spec_mult != 1.0) { pa *= p.spec_mult; pb *= p.spec_mult; }     // `normalized`
      P[k] = pa;
      P[NB + k] = pb;
    }
    group_sync(g, G);

    // ---- sparse triangular mel projection (fp64 accumulate, rounded once) + log floor (kaldi.py:630-633) ----
#pragma unroll
    for (int fr = 0; fr < 2; ++fr) {
      if (fr == 1 && !vb) break;
      const int f = fa + fr;
      const double* pf = P + fr * NB;
      for (int m = t; m < F; m += G) {
        const int st = __ldg(p.mel_start + m), cnt = __ldg(p.mel_count + m), off = __ldg(p.mel_off + m);
        double acc = 0.0;
        for (int i = 0; i < cnt; ++i) acc = fma(pf[st + i], (double)__ldg(p.mel_w + off + i), acc);
        float s = (float)acc;
        if (p.use_log == 1) s = logf(fmaxf(s, p.log_floor));                       // kaldi.py:633
        else if (p.use_log == 2) s = p.db_mult * log10f(fmaxf(s, p.log_floor));   // amplitude_to_DB, functional.py:389-391
        else if (p.use_log == 3) s = logf(s + p.log_floor);                        // MFCC(log_mels=True), transforms MFCC.forward
        vmax = fmaxf(vmax, s);
        p.feats[((size_t)b * p.T + f) * F + m] = s;
      }
    }
    group_sync(g, G);                               // P (in the FFT buffer) is overwritten by the next pair
  }
  __syncthreads();

  if (p.cta_max) {
    // ---- MFCC mel stage: per-CTA maximum for the call-wide top_db clamp (functional.py:393-399); CMN comes after the DCT
    vmax = warp_max(vmax);
    if ((tid & 31) == 0) red[tid >> 5] = vmax;
    __syncthreads();
    if (tid == 0) {
      float m = red[0];
      for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
      p.cta_max[(size_t)b * p.nblk + blockIdx.x] = m;
    }
    return;
  }
  // ---- per-CTA column sums for the CMN mean (featurizer.py:79), fixed summation order ----
  for (int m = tid; m < F; m += 256) {
    float s = 0.f;
    for (int f = f0; f < f0 + p.fpb && f < p.T; ++f) s += p.feats[((size_t)b * p.T + f) * F + m];
    p.partial[((size_t)b * p.nblk + blockIdx.x) * F + m] = s;
  }
}

// MFCC tail (torchaudio MFCC.forward): clamp the dB mel values to (max over the WHOLE call) - top_db -- torchaudio folds
// the batch axis into the clamp's channel axis, so the maximum is shared by every utterance of the call -- then
// mfcc[t, k] = sum_m mel_db[t, m] * dct[m, k] (create_dct, functional.py:640-667).  One CTA per (frame tile, utterance);
// also emits the per-CTA column sums that cmn_mask_kernel turns into the CMN mean.
__global__ void __launch_bounds__(256) mfcc_post_kernel(const __grid_constant__ MfccParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  extern __shared__ __align__(16) float sm[];
  float* dct = sm;                              // [M][K]
  float* tile = dct + p.M * p.K;                // [fpb][M]
  float* outt = tile + p.fpb * p.M;             // [fpb][K]
  float* red = outt + p.fpb * p.K;              // 8
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * p.fpb;
  float thr = -INFINITY;
  if (p.top_db >= 0.f) {
    float m = -INFINITY;
    for (int i = tid; i < p.n_max; i += 256) m = fmaxf(m, __ldg(p.cta_max + i));
    m = warp_max(m);
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    thr = m - p.top_db;
  }
  for (int i = tid; i < p.M * p.K; i += 256) dct[i] = __ldg(p.dct + i);
  for (int i = tid; i < p.fpb * p.M; i += 256) {
    const int fr = i / p.M;
    const int f = f0 + fr;
    tile[i] = f < p.T ? fmaxf(__ldg(p.mel + ((size_t)b * p.T + f) * p.M + (i - fr * p.M)), thr) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < p.fpb * p.K; i += 256) {
    const int fr = i / p.K;
    const int k = i - fr * p.K;
    const float* row = tile + fr * p.M;
    float s = 0.f;
    for (int m = 0; m < p.M; ++m) s = fmaf(row[m], dct[m * p.K + k], s);
    outt[i] = s;
    if (f0 + fr < p.T) p.feats[((size_t)b * p.T + f0 + fr) * p.K + k] = s;
  }
  __syncthreads();
  for (int k = tid; k < p.K; k += 256) {
    float s = 0.f;
    for (int fr = 0; fr < p.fpb && f0 + fr < p.T; ++fr) s += outt[fr * p.K + k];
    p.partial[((size_t)b * p.nblk + blockIdx.x) * p.K + k] = s;
  }
}

// feats[b, t, :] -= mean_t(feats[b]) over ALL T frames, then frames t >= keep[b] are zeroed (featurizer.py:79-90).
__global__ void __launch_bounds__(128) cmn_mask_kernel(float* feats, const float* partial, const int* keep, int T, int F,
                                                       int nblk, int rows_per_cta) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int b = blockIdx.y;
  const int kp = keep ? keep[b] : T;
  const int t0 = blockIdx.x * rows_per_cta;
  for (int m = threadIdx.x; m < F; m += blockDim.x) {        // F > 128 only for Spectrogram (n_fft/2 + 1 bins)
    float s = 0.f;
    for (int i = 0; i < nblk; ++i) s += partial[((size_t)b * nblk + i) * F + m];
    const float mean = s / (float)T;
    for (int t = t0; t < t0 + rows_per_cta && t < T; ++t) {
      float* q = feats + ((size_t)b * T + t) * F + m;
      *q = (t < kp) ? (*q - mean) : 0.f;
    }
  }
}

// out[0] = max(v[0..n)): the call-wide (or, sharded, the rank-wide) maximum of the per-CTA maxima of the MFCC mel stage
__global__ void __launch_bounds__(256) max_reduce_kernel(const float* v, int n, float* out) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  __shared__ float red[8];
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n; i += 256) m = fmaxf(m, v[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    out[0] = m;
  }
}

// threads per FFT group: enough for one radix-`first` pass in one sweep, a multiple of 32, at most 256
static int frontend_group_threads(int N) {
  const int first = (N % 8 == 0) ? 8 : 4;
  int G = ((N / first + 31) / 32) * 32;
  if (G < 32) G = 32;
  if (G > 256) G = 256;
  while (256 % G) G += 32;                 // G must divide the CTA (N = 400 -> 50 butterflies -> 64)
  return G;
}

// host-side pass plan: radix 8 first, then 4, 2, 5, 3 (N = 2^a 3^b 5^c checked by vp_frontend_set)
void frontend_plan(FrontendParams& p) {
  int n = p.N, k = 0;
  for (int r : {8, 4, 2, 5, 3})
    while (n % r == 0 && k < 12) { p.radix[k++] = r; n /= r; }
  p.n_pass = k;
  p.G = frontend_group_threads(p.N);
}

size_t frontend_smem_bytes(int N, int WL, int hop, int fpb) {
  const int G = frontend_group_threads(N);
  const int NG = 256 / G;
  const int span = (fpb - 1) * hop + WL;
  return sizeof(double2) * ((size_t)N + 2 * (size_t)NG * N) + sizeof(float) * (((span + 3) & ~3) + ((WL + 3) & ~3) + 2 * NG + 8 + 4);
}

// MFCC: mel stage (dB values into p.feats = the temporary mel buffer, maxima into p.cta_max), then clamp + DCT into
// m.feats and the CMN partial sums, then CMN + mask over the K cepstral coefficients.
// Dynamic shared memory above 48 KB must be opted into once per kernel; remember the largest request so far.
static cudaError_t ensure_frontend_smem(size_t smem) {
  static PerDeviceSmem once;
  if (once.need(smem)) {
    cudaError_t e = cudaFuncSetAttribute(frontend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    once.set(smem);
  }
  return cudaSuccess;
}

// MFCC stage 1 only: mel dB values + per-CTA maxima, and their maximum into max_out[0] (device) -- the scalar a sharded
// call all-reduces (MAX) across ranks before stage 2.
cudaError_t launch_frontend_mfcc_mel(const FrontendParams& p, float* max_out, cudaStream_t stream) {
  size_t smem = frontend_smem_bytes(p.N, p.WL, p.hop, p.fpb);
  cudaError_t e = ensure_frontend_smem(smem);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nblk, p.B);
  launch_pdl(frontend_kernel, grid, 256, smem, stream, p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  launch_pdl(max_reduce_kernel, 1, 256, 0, stream, p.cta_max, p.B * p.nblk, max_out);
  return cudaGetLastError();
}

// MFCC stage 2 only: clamp against m.cta_max[0..n_max) (one externally reduced scalar when n_max == 1), DCT, CMN + mask.
cudaError_t launch_frontend_mfcc_finish(const FrontendParams& p, const MfccParams& m, const int* keep, cudaStream_t stream) {
  dim3 grid(p.nblk, p.B);
  size_t smem2 = ((size_t)m.M * m.K + (size_t)m.fpb * (m.M + m.K) + 8) * sizeof(float);
  static PerDeviceSmem once;
  cudaError_t e;
  if (once.need(smem2)) {
    e = cudaFuncSetAttribute(mfcc_post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
    if (e != cudaSuccess) return e;
    once.set(smem2);
  }
  launch_pdl(mfcc_post_kernel, grid, 256, smem2, stream, m);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int rows = 64;
  dim3 g2((p.T + rows - 1) / rows, p.B);
  launch_pdl(cmn_mask_kernel, g2, 128, 0, stream, m.feats, m.partial, keep, p.T, m.K, p.nblk, rows);
  return cudaGetLastError();
}

cudaError_t launch_frontend_mfcc(const FrontendParams& p, const MfccParams& m, const int* keep, cudaStream_t stream) {
  size_t smem = frontend_smem_bytes(p.N, p.WL, p.hop, p.fpb);
  cudaError_t e = ensure_frontend_smem(smem);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nblk, p.B);
  launch_pdl(frontend_kernel, grid, 256, smem, stream, p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_frontend_mfcc_finish(p, m, keep, stream);     // clamps against all B*nblk per-CTA maxima (m.n_max)
}

cudaError_t launch_frontend(const FrontendParams& p, const int* keep, cudaStream_t stream) {
  size_t smem = frontend_smem_bytes(p.N, p.WL, p.hop, p.fpb);
  cudaError_t e = ensure_frontend_smem(smem);
  if (e != cudaSuccess) return e;
  dim3 grid(p.nblk, p.B);
  launch_pdl(frontend_kernel, grid, 256, smem, stream, p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int rows = 64;
  dim3 g2((p.T + rows - 1) / rows, p.B);
  launch_pdl(cmn_mask_kernel, g2, 128, 0, stream, p.feats, p.partial, keep, p.T, p.F, p.nblk, rows);
  return cudaGetLastError();
}

}  // namespace vpb
