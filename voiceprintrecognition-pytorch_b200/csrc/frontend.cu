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
// FFT: two real frames are packed into one complex length-N Stockham autosort FFT.  N = 2^a 3^b 5^c (4 | N): radix-8
// passes first, then radix 4 / 2, then generic radix-5 / radix-3 passes (torchaudio's default n_fft = 400 = 8*2*5*5);
// the pass plan comes from the host.  A group of G threads (a multiple of 32, G ~ N/8) owns one FFT and synchronises on
// its own named barrier, 256/G groups per CTA run independently.
//
// N = 256 / 512 / 1024 / 2048 (every shipped config) run frontend_kernel<N>: a thread holds its 8 points in registers
// through every pass (one radix-8 butterfly, or two radix-4 / four radix-2 ones), the window stage produces the first
// pass's operands in place, and the packed-spectrum split + power reads its own bins from the registers of the last
// pass and only the mirrored bins Z[N-k] from shared memory.  Any other N runs frontend_kernel<0>, the same arithmetic
// driven by the pass plan with every operand going through shared memory.  Both use the layouts below.
//
// SHARED-MEMORY LAYOUTS (16-byte double2 accesses are served a quarter-warp at a time: 8 lanes x 16 B = all 32 banks,
// so an access is conflict-free when its 8 lanes hit 8 different 16-byte slots mod 8, or the same slot).
//  * Exchange between passes: element i lives at slot xpad(i) = i + i/8.  A pass reads src[j + r*q] with j = the lane:
//    8 consecutive j (q a multiple of 8 for every power-of-two N) share j/8, so they hit 8 consecutive slots.  A pass
//    writes dst[(j-kk)*R + kk + m*Ns], kk = j % Ns.  Ns = 1 (first pass, R = 8): slot 9j + m, stride 9 over the lanes.
//    Ns >= 8 (8, 64, 512; 16, 40, 80, ... in the mixed-radix plans, all multiples of 8): the 8 lanes have consecutive
//    kk and share (j-kk) and i/8, so again 8 consecutive slots.  The unpadded layout had the Ns = 1 stores 8-way
//    conflicting.  Only the mixed-radix sizes whose q is not a multiple of 8 (n_fft 400: q = 50) keep a 2-way
//    conflict where a lane group straddles a pad.
//  * Last exchange of the register-resident path: Z[N/2+1 .. N-1] are stored unpadded and read back as Z[N-k] with
//    k = the lane: ascending on the store side, descending on the load side, 8 adjacent slots either way.
//  * Twiddles: twx[(Ns-1) + (r-1)*Ns + kk] = exp(-2 pi i r*kk / (Ns*R)) (built once on the host), the N-1 factors laid out so that
//    the lanes' kk are adjacent (the plain table was read at stride r*step: up to 8-way).  The radix-5 / radix-3
//    roots are a separate 8-entry table read at one address by every lane.
//
// PRECISION.  The window pipeline runs in fp32 op for op like the reference (those roundings are part of what the
// reference computes); the FFT, the power spectrum and the mel accumulation run in FP64 and are rounded to fp32 once.
// Why: the log turns the RELATIVE error of a mel energy into an absolute error, and with pre-emphasised input the
// low-frequency bins sit 30 dB below the frame's energy, so an fp32 FFT's absolute rounding error (any fp32 FFT, the
// reference's included) is ~1e-4 relative THERE.  Measured (tools/fbank_precision_study.py, 16 x 3 s of the bench input):
// torchaudio's own fp32 result is up to 6.1e-4 (log units) away from the exact value of its own formula, an fp32
// Stockham up to 4.1e-4, this kernel <= 2e-6.  The distance to the reference is therefore the REFERENCE's rounding
// error; no fp32 implementation can be closer to it than that without replicating its FFT library bit for bit.
// Every butterfly, twiddle product, power and mel sum is the same expression on the same operands in both
// instantiations, so the features do not depend on which one ran.
// Bound (DESIGN.md section 4 has the counts): at 256 x 3 s, 73 MB of HBM traffic, ~1 GFLOP of fp64 and ~3.2 GB through
// shared memory per call.  frontend_kernel<512> takes 0.285 ms there and the Fbank call, with cmn_mask_kernel, 0.307 ms
// (one H100 80GB HBM3, 700 W; the call took 0.61 ms before the layouts above): shared memory is the nearest bound, ~3x
// away; the rest is barrier and shared-memory latency at the 16 warps per SM that 128 registers allow.
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

// slot of element i in an exchange buffer (header comment: SHARED-MEMORY LAYOUTS)
__device__ __forceinline__ int xpad(int i) { return i + (i >> 3); }
static int xpad_len(int N) { return N + (N >> 3); }

// asynchronous global -> shared copy of BYTES (4, 8 or 16, both addresses aligned to it); cp_async_wait_all before use
template <int BYTES>
__device__ __forceinline__ void cp_async(void* dst, const void* src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  if (BYTES == 16) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
  else asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(d), "l"(src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// barrier over the G threads of one FFT group (G % 32 == 0; ids 1..8, id 0 is __syncthreads)
__device__ __forceinline__ void group_sync(int g, int G) { asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "r"(G) : "memory"); }

// ---- butterflies: v = inputs (twiddles applied), o[m] = output m ----
__device__ __forceinline__ void bfly8(const cd* v, cd* o) {
  const cd a0 = cadd(v[0], v[4]), a1 = csub(v[0], v[4]), a2 = cadd(v[2], v[6]), a3 = cmi(csub(v[2], v[6]));
  const cd a4 = cadd(v[1], v[5]), a5 = csub(v[1], v[5]), a6 = cadd(v[3], v[7]), a7 = cmi(csub(v[3], v[7]));
  const cd b0 = cadd(a0, a2), b2 = csub(a0, a2), b1 = cadd(a1, a3), b3 = csub(a1, a3);
  const cd b4 = cadd(a4, a6), b6 = cmi(csub(a4, a6));
  const double h = 0.70710678118654752440;
  const cd s5 = cadd(a5, a7), d5 = csub(a5, a7);
  const cd b5 = {h * (s5.x + s5.y), h * (s5.y - s5.x)};          // * (1 - i) / sqrt 2
  const cd b7 = {h * (d5.y - d5.x), -h * (d5.x + d5.y)};         // * (-1 - i) / sqrt 2
  o[0] = cadd(b0, b4); o[1] = cadd(b1, b5); o[2] = cadd(b2, b6); o[3] = cadd(b3, b7);
  o[4] = csub(b0, b4); o[5] = csub(b1, b5); o[6] = csub(b2, b6); o[7] = csub(b3, b7);
}
__device__ __forceinline__ void bfly4(const cd* v, cd* o) {
  const cd a0 = cadd(v[0], v[2]), a1 = csub(v[0], v[2]), a2 = cadd(v[1], v[3]), a3 = cmi(csub(v[1], v[3]));
  o[0] = cadd(a0, a2); o[1] = cadd(a1, a3); o[2] = csub(a0, a2); o[3] = csub(a1, a3);
}
__device__ __forceinline__ void bfly2(const cd* v, cd* o) {
  o[0] = cadd(v[0], v[1]);
  o[1] = csub(v[0], v[1]);
}
template <int R>
__device__ __forceinline__ void bfly(const cd* v, cd* o) {
  if (R == 8) bfly8(v, o);
  else if (R == 4) bfly4(v, o);
  else bfly2(v, o);
}

// radix of the pass that starts with `rem` points still to combine: frontend_plan's order for a power of two
__host__ __device__ constexpr int pow2_radix(int rem) { return rem % 8 == 0 ? 8 : (rem % 4 == 0 ? 4 : 2); }
__host__ __device__ constexpr int pow2_last_radix(int N) { return pow2_radix(N) == N ? N : pow2_last_radix(N / pow2_radix(N)); }
__host__ __device__ constexpr int pow2_passes(int N) { return N == 1 ? 0 : 1 + pow2_passes(N / pow2_radix(N)); }

// Passes Ns, Ns*R, ... of the register-resident FFT (N = 8 G; thread t holds 8 points).  On entry with Ns == 1 v holds
// x[t + r*G]; later passes load their operands from src.  Every pass but the last stores to dst in the padded layout and
// the buffers swap; the last leaves Z[t + i*G + m*Ns] in v[i*R + m] and stores the upper half unpadded.  Returns the
// buffer of that last store; the other one is free.
template <int N, int Ns>
__device__ __forceinline__ double2* fft_pow2(cd (&v)[8], double2* src, double2* dst, const double2* twx, int t, int g) {
  constexpr int G = N / 8, R = pow2_radix(N / Ns), q = N / R, nb = 8 / R;
  constexpr bool last = Ns * R == N;
  if (Ns > 1) {
#pragma unroll
    for (int i = 0; i < nb; ++i)
#pragma unroll
      for (int r = 0; r < R; ++r) v[i * R + r] = ld2(src + xpad(t + i * G + r * q));
  }
#pragma unroll
  for (int i = 0; i < nb; ++i) {
    const int j = t + i * G;
    const int kk = j & (Ns - 1);
    if (Ns > 1) {
#pragma unroll
      for (int r = 1; r < R; ++r) v[i * R + r] = cmul(v[i * R + r], ld2(twx + (Ns - 1) + (r - 1) * Ns + kk));
    }
    cd o[R];
    bfly<R>(&v[i * R], o);
    const int base = (j - kk) * R + kk;
#pragma unroll
    for (int m = 0; m < R; ++m) {
      v[i * R + m] = o[m];
      if (!last) st2(dst + xpad(base + m * Ns), o[m]);
      else if (i * G + m * Ns >= N / 2) st2(dst + j + m * Ns, o[m]);
    }
  }
  group_sync(g, G);
  if constexpr (last) return dst;
  else return fft_pow2<N, Ns * R>(v, dst, src, twx, t, g);
}

// |a|^2 and |b|^2 (or the magnitudes) of the two real frames packed as z = a + i b, from Z[k] and Z[N-k]
__device__ __forceinline__ void split_power(const FrontendParams& p, cd z, cd zn, double& pa, double& pb) {
  const double ar = 0.5 * (z.x + zn.x), ai = 0.5 * (z.y - zn.y);
  const double br = 0.5 * (z.y + zn.y), bi = -0.5 * (z.x - zn.x);
  pa = ar * ar + ai * ai;
  pb = br * br + bi * bi;
  if (p.power == 1) { pa = sqrt(pa); pb = sqrt(pb); }
  if (p.spec_mult != 1.0) { pa *= p.spec_mult; pb *= p.spec_mult; }     // `normalized`
}

// NFFT = 256 / 512 / 1024 / 2048: register-resident passes for that n_fft; NFFT = 0: any n_fft, plan-driven.
// A CTA owns p.tpc consecutive 16-frame tiles of one utterance and emits one CMN partial sum per tile.
template <int NFFT>
__global__ void __launch_bounds__(256, 2) frontend_kernel(const __grid_constant__ FrontendParams p) {
  pdl_launch_dependents();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = NFFT ? NFFT : p.N, WL = p.WL, F = p.F;
  const int G = NFFT ? NFFT / 8 : p.G;              // threads per FFT (multiple of 32)
  const int NG = 256 / G;                           // concurrent FFTs per CTA
  const int cfr = p.fpb * p.tpc;                    // frames per CTA
  const int span = (cfr - 1) * p.hop + WL;
  const int XN = N + (N >> 3);

  double2* twx = reinterpret_cast<double2*>(smem_raw);              // N: per-pass twiddles (N - 1 used)
  double2* roots = twx + N;                                         // 8: W_5^0..4, W_3^0..2
  double2* bufs = roots + 8;                                        // NG * 2 * XN: exchange buffers A, B of each group
  double* melw = reinterpret_cast<double*>(bufs + (size_t)NG * 2 * XN);   // mel_nw doubles (rounded up to x2)
  float* stage = reinterpret_cast<float*>(melw + ((p.mel_nw + 1) & ~1));  // span floats (rounded up to x4)
  float* win = stage + ((span + 3) & ~3);                           // WL
  float* fcache = win + ((WL + 3) & ~3);                            // cfr * F when p.cache: the CTA's features
  int* melidx = reinterpret_cast<int*>(fcache + (p.cache ? (size_t)cfr * F : 0));   // start[F], count[F], off[F]
  float* means = reinterpret_cast<float*>(melidx + 3 * F);          // NG * 2
  float* red = means + NG * 2;                                      // 8 floats: per-warp maxima (MFCC mel stage)

  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * cfr;
  const int g = tid / G;
  const int t = tid - g * G;
  float vmax = -INFINITY;
  const float* wv = p.wave + (size_t)b * p.L;

  // ---- stage the twiddles, window, mel bank and waveform span with asynchronous copies, all in flight together: one
  // global-memory latency per CTA instead of one per table.  The tables are immutable, so their copies start before
  // pdl_wait and overlap the tail of the kernel before this one. ----
  for (int i = tid; i < N + 8; i += 256) cp_async<16>(twx + i, p.twiddle + i);          // twx and roots are adjacent
  for (int i = tid; i < p.mel_nw; i += 256) cp_async<8>(melw + i, p.mel_w + i);
  for (int i = tid; i < WL; i += 256) cp_async<4>(win + i, p.window + i);
  for (int i = tid; i < F; i += 256) {
    cp_async<4>(melidx + i, p.mel_start + i);
    cp_async<4>(melidx + F + i, p.mel_count + i);
    cp_async<4>(melidx + 2 * F + i, p.mel_off + i);
  }
  pdl_wait();                 // first access to mutable global memory comes after this
  // the row's samples and frames: the call's, or in a ragged call the row's own (clamped to the stride and to T)
  const int L = p.lens ? min(max(p.lens[b], 0), p.L) : p.L;
  const int T = p.lens ? min(frontend_frames(p.kind, p.frame, WL, N, p.hop, p.kind ? p.pad : 0, L), p.T) : p.T;
  const int nblk = (T + p.fpb - 1) / p.fpb;
  if (p.lens) {
    if (blockIdx.x == 0 && tid == 0) p.row_T[b] = T;
    if (f0 >= T) { cp_async_wait_all(); return; }   // tiles past the row compute and read nothing
  }
  // the frame mode maps each staged sample to its source
  const int q0 = f0 * p.hop;
  int i0 = 0;
  if (p.kind == 0 && p.frame != VP_FRAME_KALDI_REFLECT && (reinterpret_cast<size_t>(wv + q0) & 15) == 0) {
    const int n4 = min(span, L - q0) >> 2;        // staged sample i is x[q0 + i]: 16-byte copies while inside the utterance
    for (int i = tid; i < n4; i += 256) cp_async<16>(stage + 4 * i, wv + q0 + 4 * i);
    i0 = n4 * 4;
  }
  for (int i = i0 + tid; i < span; i += 256) {
    int s = q0 + i;
    if (p.kind == 1) {                      // torch.stft of x zero-extended by p.pad at both ends: functional.py:112-134
      const int Lp = L + 2 * p.pad;
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
      if (s >= L) s = 2 * L - 1 - s;
    }
    stage[i] = (s >= 0 && s < L) ? __ldg(wv + s) : 0.f;
  }
  cp_async_wait_all();
  __syncthreads();

  // Every group owns the frame pairs g, g + NG, ... of the CTA's tiles and runs them start to finish on its own named
  // barrier: the groups never wait for each other inside the loop.
  const int npairs = cfr / 2;
  double2* bufA = bufs + (size_t)g * 2 * XN;
  double2* bufB = bufA + XN;
  const int NB = N / 2 + 1;
  for (int pair = g; pair < npairs; pair += NG) {
    const int fa = f0 + pair * 2;                   // frames packed as real (fa) and imaginary (fa + 1) parts
    const int oa = (fa - f0) * p.hop;
    const bool va = fa < T, vb = fa + 1 < T;
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
    auto windowed = [&](int j) -> cd {
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
      return {(double)ya, (double)yb};
    };

    // P[2][N/2+1]: the two power spectra, in whichever exchange buffer the FFT's last pass did not write
    double* P;
    if constexpr (NFFT != 0) {
      // ---- register-resident FFT: the first store goes to A, so the last lands in A when the pass count is odd ----
      cd v[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) v[r] = windowed(t + r * (NFFT / 8));
      const double2* zbuf = fft_pow2<NFFT, 1>(v, bufB, bufA, twx, t, g);
      P = reinterpret_cast<double*>(zbuf == bufA ? bufB : bufA);
      // ---- split the packed spectrum, power in fp64 (kaldi.py:616-618): Z[k] from the registers, Z[N-k] from zbuf ----
      constexpr int LR = pow2_last_radix(NFFT), LNs = NFFT / LR;
#pragma unroll
      for (int i = 0; i < 8 / LR; ++i)
#pragma unroll
        for (int m = 0; m < LR; ++m) {
          constexpr int Gc = NFFT / 8;
          const int kb = i * Gc + m * LNs;           // v[i * LR + m] = Z[t + kb]
          if (kb < NFFT / 2 || (kb == NFFT / 2 && t == 0)) {
            const int k = t + kb;
            const cd z = v[i * LR + m];
            const cd zn = (k == 0 || kb == NFFT / 2) ? z : ld2(zbuf + (NFFT - k));
            double pa, pb;
            split_power(p, z, zn, pa, pb);
            P[k] = pa;
            P[NB + k] = pb;
          }
        }
    } else {
      for (int j = t; j < N; j += G) st2(bufA + xpad(j), windowed(j));
      group_sync(g, G);
      // ---- Stockham autosort FFT in fp64, pass plan from the host (radix 8 / 4 / 2, then 5 / 3) ----
      double2* src = bufA;
      double2* dst = bufB;
      int Ns = 1;
      for (int ps = 0; ps < p.n_pass; ++ps) {
        const int R = p.radix[ps];
        const int q = N / R;
        const bool pow2 = (Ns & (Ns - 1)) == 0;
        for (int j = t; j < q; j += G) {
          const int kk = pow2 ? (j & (Ns - 1)) : (j % Ns);
          const int base = (j - kk) * R + kk;
          const double2* tq = twx + (Ns - 1) + kk - Ns;      // tq[r * Ns] = twiddle[r * kk * N / (Ns * R)]
          if (R == 8 || R == 4 || R == 2) {
            cd v[8], o[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)
              if (r < R) {
                v[r] = ld2(src + xpad(j + r * q));
                if (r > 0 && Ns > 1) v[r] = cmul(v[r], ld2(tq + r * Ns));
              }
            if (R == 8) bfly8(v, o);
            else if (R == 4) bfly4(v, o);
            else bfly2(v, o);
#pragma unroll
            for (int m = 0; m < 8; ++m)
              if (m < R) st2(dst + xpad(base + m * Ns), o[m]);
          } else {
            // generic odd radix (5 or 3): out[m] = sum_r v[r] * W_R^(r m)
            const double2* wr = roots + (R == 5 ? 0 : 5);
            cd v[5];
#pragma unroll
            for (int r = 0; r < 5; ++r)
              if (r < R) {
                v[r] = ld2(src + xpad(j + r * q));
                if (r > 0 && Ns > 1) v[r] = cmul(v[r], ld2(tq + r * Ns));
              }
#pragma unroll
            for (int m = 0; m < 5; ++m)
              if (m < R) {
                cd acc = v[0];
#pragma unroll
                for (int r = 1; r < 5; ++r)
                  if (r < R) acc = cadd(acc, cmul(v[r], ld2(wr + (r * m) % R)));
                st2(dst + xpad(base + m * Ns), acc);
              }
          }
        }
        group_sync(g, G);
        double2* tmp = src; src = dst; dst = tmp;
        Ns *= R;
      }
      // ---- split the packed spectrum, power in fp64 (kaldi.py:616-618) ----
      P = reinterpret_cast<double*>(dst);
      for (int k = t; k < NB; k += G) {
        double pa, pb;
        split_power(p, ld2(src + xpad(k)), ld2(src + xpad(k == 0 ? 0 : N - k)), pa, pb);
        P[k] = pa;
        P[NB + k] = pb;
      }
    }
    group_sync(g, G);

    // ---- sparse triangular mel projection (fp64 accumulate, rounded once) + log floor (kaldi.py:630-633): the 2 F
    // outputs of the frame pair over the G threads ----
    auto emit = [&](int o, double acc) {            // output o of the pair: frame o / F, bin o % F
      const int fr = o >= F, m = o - fr * F;
      float s = (float)acc;
      if (p.use_log == 1) s = logf(fmaxf(s, p.log_floor));                       // kaldi.py:633
      else if (p.use_log == 2) s = p.db_mult * log10f(fmaxf(s, p.log_floor));   // amplitude_to_DB, functional.py:389-391
      else if (p.use_log == 3) s = logf(s + p.log_floor);                        // MFCC(log_mels=True), transforms MFCC.forward
      vmax = fmaxf(vmax, s);
      p.feats[((size_t)b * p.T + fa + fr) * F + m] = s;
      if (p.cache) fcache[(size_t)(fa + fr - f0) * F + m] = s;
    };
    // Inside a bin the order i = 0 .. cnt-1 is the result's.  With several outputs per thread (Fbank-80: 160 on 64
    // threads, short chains) four of them run interleaved; with at most one per thread (64 mel bins at n_fft 1024: long
    // chains) the plain loop pipelines its loads better, and the plan-driven kernel has no registers to spare for more.
    constexpr int MU = 4;
    if (!frontend_mel_chains(NFFT, F, G)) {
      for (int o = t; o < 2 * F && (o < F || vb); o += G) {
        const int fr = o >= F, m = o - fr * F;
        const double* pf = P + fr * NB + melidx[m];
        const double* wf = melw + melidx[2 * F + m];
        const int cnt = melidx[F + m];
        double acc = 0.0;
        for (int i = 0; i < cnt; ++i) acc = fma(pf[i], wf[i], acc);
        emit(o, acc);
      }
    } else {
      for (int o0 = t; o0 < 2 * F; o0 += MU * G) {
        const double* pf[MU];
        const double* wf[MU];
        int cnt[MU], cmax = 0;
        double acc[MU];
#pragma unroll
        for (int u = 0; u < MU; ++u) {
          const int o = o0 + u * G, fr = o >= F;
          const bool live = o < 2 * F && (!fr || vb);
          const int m = live ? o - fr * F : 0;
          pf[u] = P + fr * NB + melidx[m];
          wf[u] = melw + melidx[2 * F + m];
          cnt[u] = live ? melidx[F + m] : 0;
          cmax = max(cmax, cnt[u]);
          acc[u] = 0.0;
        }
        for (int i = 0; i < cmax; ++i)
#pragma unroll
          for (int u = 0; u < MU; ++u)
            if (i < cnt[u]) acc[u] = fma(pf[u][i], wf[u][i], acc[u]);
#pragma unroll
        for (int u = 0; u < MU; ++u) {
          const int o = o0 + u * G;
          if (o < 2 * F && (o < F || vb)) emit(o, acc[u]);
        }
      }
    }
    // P is in A when the pass count is even, and the next pair's first pass writes A without a barrier before it
    if (NFFT == 0 || pow2_passes(NFFT ? NFFT : 1) % 2 == 0) group_sync(g, G);
  }
  __syncthreads();

  const int blk0 = blockIdx.x * p.tpc;              // the CTA's first 16-frame tile
  if (p.cta_max) {
    // ---- MFCC mel stage: the CTA's maximum, for every tile it owns, for the top_db clamp (functional.py:393-399)
    // against the call's maximum, or the row's in a ragged call; CMN comes after the DCT
    vmax = warp_max(vmax);
    if ((tid & 31) == 0) red[tid >> 5] = vmax;
    __syncthreads();
    if (tid < p.tpc && blk0 + tid < nblk) {
      float m = red[0];
      for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
      p.cta_max[(size_t)b * p.nblk + blk0 + tid] = m;
    }
    return;
  }
  // ---- per-tile column sums for the CMN mean (featurizer.py:79), fixed summation order; from the on-chip copy of the
  // features when it fits, else from what this CTA wrote ----
  for (int i = tid; i < p.tpc * F; i += 256) {
    const int ti = i / F, m = i - ti * F;
    if (blk0 + ti >= nblk) break;
    const int fb = f0 + ti * p.fpb;
    float s = 0.f;
    for (int f = fb; f < fb + p.fpb && f < T; ++f)
      s += p.cache ? fcache[(size_t)(f - f0) * F + m] : p.feats[((size_t)b * p.T + f) * F + m];
    p.partial[((size_t)b * p.nblk + blk0 + ti) * F + m] = s;
  }
}

// MFCC tail (torchaudio MFCC.forward): clamp the dB mel values to (max over the WHOLE call) - top_db -- torchaudio folds
// the batch axis into the clamp's channel axis, so the maximum is shared by every utterance of the call; a ragged call
// (p.row_T) featurizes each row as a call of its own, so a row is clamped against its own tiles' maxima -- then
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
  const int T = p.row_T ? p.row_T[b] : p.T;         // frames of the row (its stride stays p.T)
  if (f0 >= T) return;                              // a tile past a ragged row
  float thr = -INFINITY;
  if (p.top_db >= 0.f) {
    const float* mx = p.row_T ? p.cta_max + (size_t)b * p.nblk : p.cta_max;
    const int n_max = p.row_T ? (T + p.fpb - 1) / p.fpb : p.n_max;
    float m = -INFINITY;
    for (int i = tid; i < n_max; i += 256) m = fmaxf(m, __ldg(mx + i));
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
    tile[i] = f < T ? fmaxf(__ldg(p.mel + ((size_t)b * p.T + f) * p.M + (i - fr * p.M)), thr) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < p.fpb * p.K; i += 256) {
    const int fr = i / p.K;
    const int k = i - fr * p.K;
    const float* row = tile + fr * p.M;
    float s = 0.f;
    for (int m = 0; m < p.M; ++m) s = fmaf(row[m], dct[m * p.K + k], s);
    outt[i] = s;
    if (f0 + fr < T) p.feats[((size_t)b * p.T + f0 + fr) * p.K + k] = s;
  }
  __syncthreads();
  for (int k = tid; k < p.K; k += 256) {
    float s = 0.f;
    for (int fr = 0; fr < p.fpb && f0 + fr < T; ++fr) s += outt[fr * p.K + k];
    p.partial[((size_t)b * p.nblk + blockIdx.x) * p.K + k] = s;
  }
}

// feats[b, t, :] -= mean_t(feats[b]) over ALL T frames, then frames t >= keep[b] are zeroed (featurizer.py:79-90).
// Ragged call (row_T non-null): row b's mean is over its own row_T[b] frames (the first row_T[b] / fpb tiles' partial
// sums) and frames t >= row_T[b] are zeroed -- collate_fn's zero padding of a singly featurized utterance.
__global__ void __launch_bounds__(128) cmn_mask_kernel(float* feats, const float* partial, const int* keep, int T, int F,
                                                       int nblk, int rows_per_cta, const int* row_T, int fpb) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int b = blockIdx.y;
  const int Tb = row_T ? row_T[b] : T;
  const int nb = row_T ? (Tb + fpb - 1) / fpb : nblk;
  const int kp = keep ? keep[b] : Tb;
  const int t0 = blockIdx.x * rows_per_cta;
  for (int m = threadIdx.x; m < F; m += blockDim.x) {        // F > 128 only for Spectrogram (n_fft/2 + 1 bins)
    float s = 0.f;
    for (int i = 0; i < nb; ++i) s += partial[((size_t)b * nblk + i) * F + m];
    const float mean = s / (float)Tb;
    const int t1 = min(t0 + rows_per_cta, T);
    for (int tb = t0; tb < t1; tb += 16) {                   // 16 rows in flight: all their loads, then their stores
      float v[16];
#pragma unroll
      for (int u = 0; u < 16; ++u)
        if (tb + u < t1 && tb + u < kp) v[u] = feats[((size_t)b * T + tb + u) * F + m];
#pragma unroll
      for (int u = 0; u < 16; ++u)
        if (tb + u < t1) feats[((size_t)b * T + tb + u) * F + m] = (tb + u < kp) ? (v[u] - mean) : 0.f;
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

// radix 8 first, then 4, 2, 5, 3 (N = 2^a 3^b 5^c checked by vp_frontend_set); returns the number of passes
static int plan_radices(int N, int* radix) {
  int n = N, k = 0;
  for (int r : {8, 4, 2, 5, 3})
    while (n % r == 0 && k < 12) { radix[k++] = r; n /= r; }
  return k;
}

// The device twiddle table (FrontendParams::twiddle), N + 8 entries, from tw[k] = exp(-2 pi i k / N): the pass that starts
// at sub-transform length Ns with radix R owns out[(Ns-1) + (r-1)*Ns + kk] = tw[r * kk * N / (Ns * R)] for r = 1 .. R-1,
// kk < Ns (adjacent lanes read adjacent entries); out[N-1] is unused; out[N .. N+4] = W_5^k, out[N+5 .. N+7] = W_3^k.
void frontend_twiddle_table(int N, const double2* tw, double2* out) {
  int radix[12];
  const int n_pass = plan_radices(N, radix);
  int Ns = 1;
  for (int ps = 0; ps < n_pass; Ns *= radix[ps++])
    for (int r = 1; r < radix[ps]; ++r)
      for (int kk = 0; kk < Ns; ++kk) out[(Ns - 1) + (r - 1) * Ns + kk] = tw[r * kk * (N / (Ns * radix[ps]))];
  out[N - 1] = make_double2(0.0, 0.0);
  for (int k = 0; k < 8; ++k) {
    const int R = k < 5 ? 5 : 3, e = k < 5 ? k : k - 5;
    out[N + k] = (N % R == 0) ? tw[e * (N / R)] : make_double2(0.0, 0.0);
  }
}

// dynamic shared memory of one CTA that owns `tpc` 16-frame tiles (frontend_kernel's carve-up)
static size_t frontend_smem_bytes(const FrontendParams& p, int tpc, bool cache) {
  const int NG = 256 / p.G;
  const int cfr = p.fpb * tpc;
  const int span = (cfr - 1) * p.hop + p.WL;
  return sizeof(double2) * ((size_t)p.N + 8 + 2 * (size_t)NG * xpad_len(p.N)) + sizeof(double) * ((p.mel_nw + 1) & ~1) +
         sizeof(float) * (((span + 3) & ~3) + ((p.WL + 3) & ~3) + (cache ? (size_t)cfr * p.F : 0) + 3 * p.F + 2 * NG + 8);
}

// Host-side plan.  Passes: radix 8 first, then 4, 2, 5, 3 (N = 2^a 3^b 5^c checked by vp_frontend_set).  CTA shape: the
// kernel is held to 128 registers, i.e. two CTAs of 256 threads per SM, so a CTA takes as many 16-frame tiles (4, 2 or
// 1: the twiddle / window / mel-bank set-up is paid once per CTA) as leave it within half an SM's shared memory,
// on-chip copy of its features included.  The large n_fft / hop / bin-count combinations that exceed that run one tile
// per CTA and drop the on-chip copy if it does not fit the 227 KB a CTA may have.
void frontend_plan(FrontendParams& p, bool mfcc_mel) {
  p.n_pass = plan_radices(p.N, p.radix);
  p.G = frontend_group_threads(p.N);
  const size_t half_sm = (228 * 1024 - 2 * 1024) / 2, cta_max = 227 * 1024;
  const bool want = !mfcc_mel;                       // the MFCC mel stage emits maxima, no column sums
  p.tpc = 1;
  p.cache = want && frontend_smem_bytes(p, 1, true) <= cta_max;
  for (int tpc : {4, 2})
    if (tpc <= p.nblk && frontend_smem_bytes(p, tpc, want) <= half_sm) { p.tpc = tpc; p.cache = want; break; }
}

// Dynamic shared memory above 48 KB must be opted into once per kernel; remember the largest request so far.
template <int NFFT>
static cudaError_t launch_frontend_kernel_n(const FrontendParams& p, size_t smem, cudaStream_t stream) {
  static PerDeviceSmem once;
  if (once.need(smem)) {
    cudaError_t e = cudaFuncSetAttribute(frontend_kernel<NFFT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    once.set(smem);
  }
  dim3 grid(frontend_grid_x(p), p.B);
  launch_pdl(frontend_kernel<NFFT>, grid, 256, smem, stream, p);
  return cudaGetLastError();
}

// the instantiation for p.N: register-resident passes for the power-of-two sizes, the plan-driven kernel for the rest
static cudaError_t launch_frontend_kernel(const FrontendParams& p, cudaStream_t stream) {
  const size_t smem = frontend_smem_bytes(p, p.tpc, p.cache);
  switch (frontend_instantiation(p.N)) {
    case 256: return launch_frontend_kernel_n<256>(p, smem, stream);
    case 512: return launch_frontend_kernel_n<512>(p, smem, stream);
    case 1024: return launch_frontend_kernel_n<1024>(p, smem, stream);
    case 2048: return launch_frontend_kernel_n<2048>(p, smem, stream);
    default: return launch_frontend_kernel_n<0>(p, smem, stream);
  }
}

// MFCC stage 1 only: mel dB values + per-CTA maxima, and their maximum into max_out[0] (device) -- the scalar a sharded
// call all-reduces (MAX) across ranks before stage 2.
cudaError_t launch_frontend_mfcc_mel(const FrontendParams& p, float* max_out, cudaStream_t stream) {
  cudaError_t e = launch_frontend_kernel(p, stream);
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
  launch_pdl(cmn_mask_kernel, g2, 128, 0, stream, m.feats, m.partial, keep, p.T, m.K, p.nblk, rows, m.row_T, p.fpb);
  return cudaGetLastError();
}

// MFCC: mel stage (dB values into p.feats = the temporary mel buffer, maxima into p.cta_max), then clamp + DCT into
// m.feats and the CMN partial sums, then CMN + mask over the K cepstral coefficients.
cudaError_t launch_frontend_mfcc(const FrontendParams& p, const MfccParams& m, const int* keep, cudaStream_t stream) {
  cudaError_t e = launch_frontend_kernel(p, stream);
  if (e != cudaSuccess) return e;
  return launch_frontend_mfcc_finish(p, m, keep, stream);     // clamps against all B*nblk per-CTA maxima (m.n_max)
}

cudaError_t launch_frontend(const FrontendParams& p, const int* keep, cudaStream_t stream) {
  cudaError_t e = launch_frontend_kernel(p, stream);
  if (e != cudaSuccess) return e;
  const int rows = 64;
  dim3 g2((p.T + rows - 1) / rows, p.B);
  launch_pdl(cmn_mask_kernel, g2, 128, 0, stream, p.feats, p.partial, keep, p.T, p.F, p.nblk, rows, p.row_T, p.fpb);
  return cudaGetLastError();
}

}  // namespace vpb
