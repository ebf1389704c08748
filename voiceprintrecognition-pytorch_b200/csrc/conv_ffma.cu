// Exact-fp32 implicit-GEMM convolution (FFMA pipe) with fused gather prologue and epilogue.
//
// Replaces, per layer, the reference's  F.pad(reflect) -> nn.Conv1d/Conv2d -> ReLU/BN/...  op chains
// (mvector/models/utils.py:39-138, campplus.py:41-111,219-255, resnet_se.py:23-44, eres2net.py:85-108) with ONE kernel:
//   out[m, n] = epi( sum_k A(m, k) * W[n, k] ),  m = (b, to, fo), k = (kt, kf, ci)
// A is gathered on the fly from the channel-last activation map (no im2col / no padded copy / no concat copy).
// This is the bit-faithful fp32 engine: used for layers that are not tensor-core shaped (small N/K, tiny M) and as the
// on-device cross-check of the tensor-core engine (conv_tc.cu).
//
// Tiling: CTA = 256 threads, 128 (M) x BN (N) x 16 (K) tiles, register-prefetch double buffering, 8 x TN micro-tile.
#include "kernels.cuh"

namespace vpb {

constexpr int BM = 128;
constexpr int BK = 16;
constexpr int LDS_PAD = 4;

template <int BN>
__global__ void __launch_bounds__(256, 2) conv_ffma_kernel(const __grid_constant__ ConvParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  constexpr int TN = BN / 16;           // columns per thread: 8, 4 or 2
  constexpr int LDA = BM + LDS_PAD;
  constexpr int LDB = BN + LDS_PAD;
  __shared__ __align__(16) float As[2][BK][LDA];
  __shared__ __align__(16) float Bs[2][BK][LDB];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- loader mapping: 4 lanes cover one row's 16 K-floats (64 B) ----
  const int kq = tid & 3;
  const int lr = tid >> 2;              // 0..63
  RowInfo rowA0 = decode_row(p, m0 + lr);
  RowInfo rowA1 = decode_row(p, m0 + lr + 64);
  constexpr int B_LOADS = (BN >= 128) ? 2 : 1;
  const bool b_active = (BN >= 64) || (lr < BN);

  float4 ra0, ra1, rb[B_LOADS];
  auto load_tiles = [&](int k0) {
    int k = k0 + kq * 4;
    ra0 = gather_a4(p, rowA0, k);
    ra1 = gather_a4(p, rowA1, k);
#pragma unroll
    for (int i = 0; i < B_LOADS; ++i) {
      int n = n0 + lr + i * 64;
      rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b_active && n < p.N && k < p.K)
        rb[i] = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)n * p.w_ld + k));
    }
  };
  auto store_tiles = [&](int buf) {
    float* a = &As[buf][kq * 4][0];
    a[0 * LDA + lr] = ra0.x; a[1 * LDA + lr] = ra0.y; a[2 * LDA + lr] = ra0.z; a[3 * LDA + lr] = ra0.w;
    a[0 * LDA + lr + 64] = ra1.x; a[1 * LDA + lr + 64] = ra1.y; a[2 * LDA + lr + 64] = ra1.z; a[3 * LDA + lr + 64] = ra1.w;
    if (b_active) {
      float* b = &Bs[buf][kq * 4][0];
#pragma unroll
      for (int i = 0; i < B_LOADS; ++i) {
        b[0 * LDB + lr + i * 64] = rb[i].x; b[1 * LDB + lr + i * 64] = rb[i].y;
        b[2 * LDB + lr + i * 64] = rb[i].z; b[3 * LDB + lr + i * 64] = rb[i].w;
      }
    }
  };

  // ---- compute mapping: 16 x 16 threads, rows {ty*4..+3, 64+ty*4..+3}, cols per TN ----
  const int tx = tid & 15;
  const int ty = tid >> 4;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (p.K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      if constexpr (TN == 8) {
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
      } else if constexpr (TN == 4) {
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      } else {
        float2 b0 = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
        b[0] = b0.x; b[1] = b0.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- fused epilogue ----
  float tmax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
    const int urow = urow_of(p, m);
    float* orow = p.dst + (size_t)m * p.out_ld + p.out_coff;
    if constexpr (TN == 8) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n0 + h * 64 + tx * 4;
        if (n + 3 < p.N) {
          float4 o;
          o.x = epilogue1(p, acc[i][h * 4 + 0], m, n + 0, urow);
          o.y = epilogue1(p, acc[i][h * 4 + 1], m, n + 1, urow);
          o.z = epilogue1(p, acc[i][h * 4 + 2], m, n + 2, urow);
          o.w = epilogue1(p, acc[i][h * 4 + 3], m, n + 3, urow);
          *reinterpret_cast<float4*>(orow + n) = o;
          sum_add4(p, m, n, o);
          tmax = amax4(tmax, o);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (n + j < p.N) {
              const float y = epilogue1(p, acc[i][h * 4 + j], m, n + j, urow);
              orow[n + j] = y;
              sum_add1(p, m, n + j, y);
              tmax = fmaxf(tmax, fabsf(y));
            }
        }
      }
    } else {
      const int n = n0 + tx * TN;
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (n + j < p.N) {
          const float y = epilogue1(p, acc[i][j], m, n + j, urow);
          orow[n + j] = y;
          sum_add1(p, m, n + j, y);
          tmax = fmaxf(tmax, fabsf(y));
        }
    }
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

// ---------------------------------------------------------------------------------------------------------------
// Small-M linear layers (SE excitation MLPs, the ASP per-utterance bias, the final embedding FC, CAM++ context MLPs):
// M <= 1024 rows but K up to 3072.  The tiled kernel above would run them on a handful of CTAs with a long serial K
// loop; here one warp owns (row m, 32 output columns), lanes stride over K with coalesced 128 B loads of x and of
// each weight row, then a fixed-order butterfly reduction -> deterministic.  grid = (ceil(N/32), ceil(M/8)).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) linear_small_m_kernel(const __grid_constant__ ConvParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  // W tile [32 output columns][128 K] staged in shared memory once per CTA and K chunk, shared by the CTA's 8 rows
  __shared__ __align__(16) float ws[32][132];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int m = blockIdx.y * 8 + wid;
  const int n0 = blockIdx.x * 32;
  const bool mok = m < p.M;
  const float* x = p.src + (size_t)(mok ? m : 0) * p.in_ld + p.in_coff;   // pointwise, stride 1: source row == output row
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += 128) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {                       // 32 rows x 32 float4 = 1024 float4, 4 per thread, coalesced rows
      const int idx = threadIdx.x + i * 256;
      const int j = idx >> 5, c = (idx & 31) * 4;
      float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n0 + j < p.N && k0 + c < p.K) wv = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)(n0 + j) * p.w_ld + k0 + c));
      *reinterpret_cast<float4*>(&ws[j][c]) = wv;
    }
    __syncthreads();
    const int k = k0 + lane * 4;
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mok && k < p.K) xv = __ldg(reinterpret_cast<const float4*>(x + k));
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float4 wv = *reinterpret_cast<const float4*>(&ws[j][lane * 4]);
      acc[j] = fmaf(xv.x, wv.x, acc[j]);
      acc[j] = fmaf(xv.y, wv.y, acc[j]);
      acc[j] = fmaf(xv.z, wv.z, acc[j]);
      acc[j] = fmaf(xv.w, wv.w, acc[j]);
    }
  }
  // transpose-reduce: after the butterfly lane j holds the total of column j (fixed order -> deterministic)
  float mine = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float t = warp_sum(acc[j]);
    if (lane == j) mine = t;
  }
  const int n = n0 + lane;
  float tmax = 0.f;
  if (mok && n < p.N) {
    const float y = epilogue1(p, mine, m, n, urow_of(p, m));
    p.dst[(size_t)m * p.out_ld + p.out_coff + n] = y;
    sum_add1(p, m, n, y);
    tmax = fabsf(y);
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

static bool small_m_ok(const ConvParams& p) {
  return p.M <= 1024 && p.KT == 1 && p.KF == 1 && p.sT == 1 && p.sF == 1 && p.padT == 0 && p.padF == 0 &&
         p.src2_mode == VP_SRC2_NONE && p.pre_s == nullptr && p.Tin == p.Tout && p.Fin == p.Fout && (p.K & 3) == 0;
}

cudaError_t launch_conv_ffma(const ConvParams& p, cudaStream_t stream) {
  dim3 block(256);
  if (small_m_ok(p)) {
    dim3 grid((p.N + 31) / 32, (p.M + 7) / 8);
    launch_pdl(linear_small_m_kernel, grid, block, 0, stream, p);
    return cudaGetLastError();
  }
  if (p.N > 64) {
    dim3 grid((p.M + BM - 1) / BM, (p.N + 127) / 128);
    launch_pdl(conv_ffma_kernel<128>, grid, block, 0, stream, p);
  } else if (p.N > 32) {
    dim3 grid((p.M + BM - 1) / BM, 1);
    launch_pdl(conv_ffma_kernel<64>, grid, block, 0, stream, p);
  } else {
    dim3 grid((p.M + BM - 1) / BM, 1);
    launch_pdl(conv_ffma_kernel<32>, grid, block, 0, stream, p);
  }
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// KTxKF (<= 7x7) strided conv2d with a single input channel on the feature map (the stem of the 2-D backbones):
//   F.relu(bn1(conv1(x.unsqueeze(1))))  campplus.py:284, resnet_se.py:131-133, eres2net.py:243 (3x3, stride 1) and
//   res2net.py:100 (7x7, stride 3, padding 1)
// in: feats [B, T, F] (one channel), out: [B, T', F', C] channel-last.  w: [C][kt][kf] (BN folded by the host), bias [C].
// One thread per output position x 4 output channels.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv_c1_kernel(const __grid_constant__ ConvParams p) {
  pdl_launch_dependents();
  pdl_wait();                 // first access to mutable global memory comes after this
  const int groups = p.N >> 2;
  const long long total = (long long)p.M * groups;
  const int taps = p.KT * p.KF;
  float tmax = 0.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    const int m = (int)(idx / groups);
    RowInfo r = decode_row(p, m);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const float* w0 = p.w + (size_t)(g * 4) * p.w_ld;
    for (int kt = 0; kt < p.KT; ++kt) {
      const int ti = r.t0 + kt * p.dT;
      if (ti < 0 || ti >= p.Tin) continue;
      for (int kf = 0; kf < p.KF; ++kf) {
        const int fi = r.f0 + kf * p.dF;
        if (fi < 0 || fi >= p.Fin) continue;
        const float x = __ldg(p.src + ((size_t)r.base + (size_t)ti * p.Fin + fi) * p.in_ld + p.in_coff);
        const int k = kt * p.KF + kf;
        a0 = fmaf(x, __ldg(w0 + k), a0);
        a1 = fmaf(x, __ldg(w0 + p.w_ld + k), a1);
        a2 = fmaf(x, __ldg(w0 + 2 * p.w_ld + k), a2);
        a3 = fmaf(x, __ldg(w0 + 3 * p.w_ld + k), a3);
      }
    }
    (void)taps;
    const int urow = urow_of(p, m);
    const int n = g * 4;
    const float4 o = make_float4(epilogue1(p, a0, m, n, urow), epilogue1(p, a1, m, n + 1, urow), epilogue1(p, a2, m, n + 2, urow),
                                 epilogue1(p, a3, m, n + 3, urow));
    *reinterpret_cast<float4*>(p.dst + (size_t)m * p.out_ld + p.out_coff + n) = o;
    tmax = amax4(tmax, o);
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

// Wide variant for the usual stems (N = 16 / 32 / 64 output channels, plain bias -> act -> affine -> act2 epilogue): one
// thread owns TWO output positions x ALL N channels.  The transposed weights [tap][N] sit in shared memory and are read
// as broadcast float4s (one LDS.128 feeds 8 FMAs), every input sample is loaded once per position, and a thread writes
// 2 x N contiguous floats, so a warp's stores cover 64 x N x 4 contiguous bytes.  ~13 instructions per output instead of
// ~25 for the generic kernel above, whose one-thread-per-4-channels layout re-loads every sample N/4 times.
template <int NQ>      // N / 4
__global__ void __launch_bounds__(256) conv_c1_wide_kernel(const __grid_constant__ ConvParams p) {
  pdl_launch_dependents();
  __shared__ float4 ws[49 * NQ];         // [tap][NQ]
  __shared__ float4 bs[NQ], ss[NQ], hs[NQ];
  const int taps = p.KT * p.KF;
  for (int i = threadIdx.x; i < taps * NQ; i += 256) {
    const int k = i / NQ, q = i - k * NQ;
    ws[i] = make_float4(__ldg(p.w + (size_t)(q * 4 + 0) * p.w_ld + k), __ldg(p.w + (size_t)(q * 4 + 1) * p.w_ld + k),
                        __ldg(p.w + (size_t)(q * 4 + 2) * p.w_ld + k), __ldg(p.w + (size_t)(q * 4 + 3) * p.w_ld + k));
  }
  for (int q = threadIdx.x; q < NQ; q += 256) {
    bs[q] = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    ss[q] = p.post_s ? __ldg(reinterpret_cast<const float4*>(p.post_s) + q) : make_float4(1.f, 1.f, 1.f, 1.f);
    hs[q] = p.post_s ? __ldg(reinterpret_cast<const float4*>(p.post_h) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  pdl_wait();                            // weights / bias are immutable; the feature map and the output are not
  float tmax = 0.f;
  const long long pairs = ((long long)p.M + 1) >> 1;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < pairs; idx += (long long)gridDim.x * blockDim.x) {
    float4 acc[2][NQ];
    RowInfo r[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      r[u] = decode_row(p, (int)(2 * idx + u));
#pragma unroll
      for (int q = 0; q < NQ; ++q) acc[u][q] = bs[q];
    }
    for (int kt = 0; kt < p.KT; ++kt)
      for (int kf = 0; kf < p.KF; ++kf) {
        float x[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int ti = r[u].t0 + kt * p.dT, fi = r[u].f0 + kf * p.dF;
          x[u] = 0.f;
          if (r[u].valid && (unsigned)ti < (unsigned)p.Tin && (unsigned)fi < (unsigned)p.Fin)
            x[u] = __ldg(p.src + ((size_t)r[u].base + (size_t)ti * p.Fin + fi) * p.in_ld + p.in_coff);
        }
        const float4* wk = ws + (kt * p.KF + kf) * NQ;
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
          const float4 w = wk[q];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            acc[u][q].x = fmaf(x[u], w.x, acc[u][q].x); acc[u][q].y = fmaf(x[u], w.y, acc[u][q].y);
            acc[u][q].z = fmaf(x[u], w.z, acc[u][q].z); acc[u][q].w = fmaf(x[u], w.w, acc[u][q].w);
          }
        }
      }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (!r[u].valid) continue;
      float4* o = reinterpret_cast<float4*>(p.dst + (size_t)(2 * idx + u) * p.out_ld + p.out_coff);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        float4 v = acc[u][q];
        v.x = apply_act(v.x, p.act); v.y = apply_act(v.y, p.act); v.z = apply_act(v.z, p.act); v.w = apply_act(v.w, p.act);
        v.x = fmaf(v.x, ss[q].x, hs[q].x); v.y = fmaf(v.y, ss[q].y, hs[q].y);
        v.z = fmaf(v.z, ss[q].z, hs[q].z); v.w = fmaf(v.w, ss[q].w, hs[q].w);
        v.x = apply_act(v.x, p.act2); v.y = apply_act(v.y, p.act2); v.z = apply_act(v.z, p.act2); v.w = apply_act(v.w, p.act2);
        o[q] = v;
        tmax = amax4(tmax, v);
      }
    }
  }
  if (p.amax_out) amax_commit_block(p.amax_out, tmax);
}

cudaError_t launch_conv_c1(const ConvParams& p, cudaStream_t stream) {
  // wide variant: N in {16, 32, 64}, <= 49 taps, epilogue = bias / act / affine / act2 only (what every stem uses)
  const bool plain = !p.ubias && !p.gate && !p.res && !p.sum && (p.N == 16 || p.N == 32 || p.N == 64) && p.KT * p.KF <= 49 &&
                     (p.out_ld & 3) == 0 && (p.out_coff & 3) == 0;
  if (plain) {
    const long long pairs = ((long long)p.M + 1) >> 1;
    long long blocks = (pairs + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (p.N == 16) launch_pdl(conv_c1_wide_kernel<4>, (int)blocks, 256, 0, stream, p);
    else if (p.N == 32) launch_pdl(conv_c1_wide_kernel<8>, (int)blocks, 256, 0, stream, p);
    else launch_pdl(conv_c1_wide_kernel<16>, (int)blocks, 256, 0, stream, p);
    return cudaGetLastError();
  }
  long long total = (long long)p.M * (p.N >> 2);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_pdl(conv_c1_kernel, blocks, 256, 0, stream, p);
  return cudaGetLastError();
}

}  // namespace vpb
