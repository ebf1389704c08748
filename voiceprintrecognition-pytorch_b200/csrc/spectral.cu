// Spectral stage of the diarization clustering (SpectralCluster, infer_utils/speaker_diarization.py:235-310):
//   (a) pruned cosine affinity -> symmetrised fp64 affinity -> unnormalised Laplacian L = diag(d) - S;
//   (b) Householder reduction of L to tridiagonal form, LAPACK dsytd2 (UPLO = 'L') convention, in place, fp64;
//   (c) back-transformation Z <- Q Z of a [n, k] block of tridiagonal eigenvectors.
// The small tridiagonal eigenproblem itself (2n numbers) is solved on the host (mvector/engine.py::spectral_embedding).
// Every reduction has a fixed order and no kernel uses floating-point atomics: results are bit-reproducible.
#include <cooperative_groups.h>

#include "kernels.cuh"

namespace cg = cooperative_groups;

namespace vpb {

// ---- block-wide fp64 sum in a fixed order (every thread gets the result; blockDim a multiple of 32, <= 1024) ----
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ double block_sum_d(double v, double* red /* [33] shared */) {
  v = warp_sum_d(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();                                     // red may still be read by a previous call
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    double s = lane < nw ? red[lane] : 0.0;
    s = warp_sum_d(s);
    if (lane == 0) red[32] = s;
  }
  __syncthreads();
  return red[32];
}

// =====================================================================================================================
// (a) Laplacian
// =====================================================================================================================

// Order-preserving 32-bit key of a float (-0 is folded onto +0: numpy compares them equal).
__device__ __forceinline__ unsigned f2key(float f) {
  unsigned u = __float_as_uint(f == 0.f ? 0.f : f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// One CTA per row of the fp32 affinity S [n, n] (in place): zero the n_drop smallest entries of the row, ties at the cut
// going by column index (lower indices first) -- np.argsort(kind='stable')[:n_drop] (p_pruning, :260-274).  The row is
// staged as keys in shared memory; a 4 x 8-bit radix select finds the key T of the n_drop-th smallest entry and how many
// entries equal to T must go; those are marked in index order with a block-wide exclusive scan over contiguous segments.
constexpr int PRUNE_THREADS = 512;

__global__ void __launch_bounds__(PRUNE_THREADS) prune_rows_kernel(float* __restrict__ S, int n, int n_drop) {
  extern __shared__ unsigned keys[];
  __shared__ unsigned hist[256];
  __shared__ unsigned s_sel[2];
  __shared__ int scan[PRUNE_THREADS / 32 + 1];
  pdl_launch_dependents();
  pdl_wait();
  if (n_drop <= 0) return;
  float* row = S + (size_t)blockIdx.x * n;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int j = tid; j < n; j += PRUNE_THREADS) keys[j] = f2key(row[j]);
  unsigned prefix = 0u, mask = 0u, rank = (unsigned)(n_drop - 1);     // 0-based rank of the last dropped entry
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += PRUNE_THREADS) hist[b] = 0u;
    __syncthreads();
    for (int j = tid; j < n; j += PRUNE_THREADS) {
      const unsigned k = keys[j];
      if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);    // integer counts: order independent
    }
    __syncthreads();
    if (wid == 0) {                                    // warp 0: lane l owns bins 8l .. 8l+7
      unsigned c[8], tot = 0u;
#pragma unroll
      for (int q = 0; q < 8; ++q) { c[q] = hist[lane * 8 + q]; tot += c[q]; }
      unsigned incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      unsigned excl = incl - tot;
      if (rank >= excl && rank < incl) {               // exactly one lane holds the bin of the rank-th key
        unsigned r = rank - excl;
        int b = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (b == q && r >= c[q]) { r -= c[q]; b = q + 1; }
        s_sel[0] = prefix | ((unsigned)(lane * 8 + b) << shift);
        s_sel[1] = r;
      }
    }
    __syncthreads();
    prefix = s_sel[0];
    rank = s_sel[1];
    mask |= 255u << shift;
  }
  const unsigned T = prefix;                           // key of the n_drop-th smallest entry
  const int ties = (int)rank + 1;                      // entries equal to T that are dropped (the lowest indices)
  // contiguous segment per thread: count keys == T, exclusive scan in thread order, then mark the first `ties` with key 0
  // (0 is the key of no finite float, so "key < T" becomes the drop test)
  const int seg = (n + PRUNE_THREADS - 1) / PRUNE_THREADS;
  const int j0 = min(n, tid * seg), j1 = min(n, j0 + seg);
  int cnt = 0;
  for (int j = j0; j < j1; ++j) cnt += keys[j] == T;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) scan[wid] = incl;
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int w = 0; w < PRUNE_THREADS / 32; ++w) { const int t = scan[w]; scan[w] = run; run += t; }
  }
  __syncthreads();
  int before = scan[wid] + incl - cnt;
  for (int j = j0; j < j1 && before < ties; ++j)
    if (keys[j] == T) { keys[j] = 0u; ++before; }
  __syncthreads();
  for (int j = tid; j < n; j += PRUNE_THREADS)
    if (keys[j] < T) row[j] = 0.f;
}

// L[i, j] = 0 - 0.5 * (P[i, j] + P[j, i]) in fp64 off the diagonal, 0 on it (the degrees follow).  32 x 32 tiles, the
// transposed tile through shared memory.
__global__ void __launch_bounds__(256) symmetrize_kernel(const float* __restrict__ P, double* __restrict__ L, int n) {
  __shared__ float t[32][33];
  pdl_launch_dependents();
  pdl_wait();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
  for (int r = ty; r < 32; r += 8) {                   // tile (j0.., i0..) of P, transposed into t[c][r]
    const int row = j0 + r, col = i0 + tx;
    t[tx][r] = (row < n && col < n) ? P[(size_t)row * n + col] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int i = i0 + r, j = j0 + tx;
    if (i < n && j < n) {
      const double s = 0.5 * ((double)P[(size_t)i * n + j] + (double)t[r][tx]);
      L[(size_t)i * n + j] = i == j ? 0.0 : 0.0 - s;
    }
  }
}

// d_i = sum_j |S_ij| (thread-strided partial sums, then the fixed block tree); L[i, i] = d_i - 0.
__global__ void __launch_bounds__(256) degree_kernel(double* __restrict__ L, int n) {
  __shared__ double red[33];
  pdl_launch_dependents();
  pdl_wait();
  double* row = L + (size_t)blockIdx.x * n;
  double s = 0.0;
  for (int j = threadIdx.x; j < n; j += 256) s += fabs(row[j]);
  s = block_sum_d(s, red);
  if (threadIdx.x == 0) row[blockIdx.x] = s;
}

// =====================================================================================================================
// (b) Householder tridiagonalisation (dsytd2, lower).  Step k (0 <= k <= n-3) reflects column k:
//   v_k = [0..0, 1, x / (alpha - beta)] (support k+1..n-1), beta = -sign(alpha) ||(alpha, x)||, tau_k = (beta - alpha) / beta,
//   p_k = A_k v_k on the trailing block T_k = [k+1, n)^2, w_k = tau p - (tau/2) (tau p . v) v,
//   A_{k+1} = A_k - v w' - w v' on T_k.
// Per step two launches:
//   reflect_kernel (one CTA)   reduces the pass's per-CTA partial sums into p_{k-1}, forms w_{k-1}; applies update k-1
//                              to column k (read as row k: the stored matrix is exactly symmetric), forms v_k, tau_k, d_k,
//                              e_k and writes the reflector into A[k+2:, k];
//   tridiag_pass_kernel        one sweep over T_k: applies update k-1 in place and accumulates p_k = A_k v_k.
// The rank-2 term is evaluated as v_i w_j + w_i v_j without contraction, which is the same number for (i, j) and (j, i):
// the full-storage matrix stays exactly symmetric.
// Scratch (doubles): vbuf[2][n] | wbuf[2][n] | partial[PASS_GY_MAX][n], double-buffered by step parity.
// =====================================================================================================================
constexpr int PASS_THREADS = 256;
constexpr int PASS_GY_MAX = 32;
constexpr int REFLECT_THREADS = 1024;

__device__ __forceinline__ double rank2(double vi, double wj, double wi, double vj) {
  return __dadd_rn(__dmul_rn(vi, wj), __dmul_rn(wi, vj));
}

__global__ void __launch_bounds__(REFLECT_THREADS) reflect_kernel(double* __restrict__ A, int n, int k, int gy_prev,
                                                                  double* __restrict__ scr, double* __restrict__ d,
                                                                  double* __restrict__ e, double* __restrict__ tau) {
  __shared__ double red[33];
  __shared__ double s_wk;
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x;
  const size_t nn = (size_t)n;
  double* vbuf = scr;
  double* wbuf = scr + 2 * nn;
  const double* partial = scr + 4 * nn;
  double* vprev = vbuf + ((k + 1) & 1) * nn;           // (k - 1) & 1
  double* wprev = wbuf + ((k + 1) & 1) * nn;
  double* vk = vbuf + (k & 1) * nn;
  double* Ak = A + (size_t)k * nn;                     // row k
  if (k >= 1) {                                        // w_{k-1} over T_{k-1} = [k, n)
    const double t = tau[k - 1];
    double dot = 0.0;
    for (int i = k + tid; i < n; i += REFLECT_THREADS) {
      double p = 0.0;
      for (int g = 0; g < gy_prev; ++g) p += partial[(size_t)g * nn + i];
      const double x = t * p;
      wprev[i] = x;
      dot += x * vprev[i];
    }
    dot = block_sum_d(dot, red);
    const double a = -0.5 * t * dot;
    for (int i = k + tid; i < n; i += REFLECT_THREADS) wprev[i] = wprev[i] + a * vprev[i];
    if (tid == 0) s_wk = wprev[k];
    __syncthreads();
  }
  // column k of A_k (rows k..n-1), kept in row k
  const double wk = k >= 1 ? s_wk : 0.0;              // w_{k-1}[k]; v_{k-1}[k] = 1
  double sig = 0.0;
  for (int i = k + tid; i < n; i += REFLECT_THREADS) {
    double c = Ak[i];
    if (k >= 1) c = __dsub_rn(c, rank2(vprev[i], wk, wprev[i], 1.0));
    Ak[i] = c;
    if (i >= k + 2) sig += c * c;
  }
  sig = block_sum_d(sig, red);                         // also orders the row-k writes before the reads below
  if (k >= n - 2) {                                    // last (or only) column: no reflector
    if (tid == 0) {
      d[k] = Ak[k];
      if (k == n - 2) {
        e[k] = Ak[k + 1];
        tau[k] = 0.0;
        A[(size_t)(k + 1) * nn + k] = Ak[k + 1];
        double c = A[(size_t)(k + 1) * nn + k + 1];
        if (k >= 1) c = __dsub_rn(c, rank2(vprev[k + 1], wprev[k + 1], wprev[k + 1], vprev[k + 1]));
        d[k + 1] = c;
        A[(size_t)(k + 1) * nn + k + 1] = c;
      }
    }
    return;
  }
  const double alpha = Ak[k + 1];
  double beta, t, scal;
  if (sig == 0.0) {                                    // dlarfg: x = 0 -> H = I
    beta = alpha; t = 0.0; scal = 0.0;
  } else {
    beta = -copysign(sqrt(alpha * alpha + sig), alpha);
    t = (beta - alpha) / beta;
    scal = 1.0 / (alpha - beta);
  }
  for (int i = k + 2 + tid; i < n; i += REFLECT_THREADS) {
    const double v = Ak[i] * scal;
    vk[i] = v;
    A[(size_t)i * nn + k] = v;
  }
  if (tid == 0) {
    vk[k + 1] = 1.0;
    A[(size_t)(k + 1) * nn + k] = beta;
    A[(size_t)k * nn + k] = Ak[k];
    d[k] = Ak[k];
    e[k] = beta;
    tau[k] = t;
  }
}

// One sweep over the trailing block T_k = [k+1, n)^2: (PREV) A -= v w' + w v' of step k-1, then partial[by][j] =
// sum over this CTA's rows i of A_ij v_k[i] (= (A v_k)_j by symmetry).  Threads own columns (coalesced rows), CTAs
// tile rows in blockIdx.y; the reflect kernel adds the partial sums in blockIdx.y order.
template <bool PREV>
__global__ void __launch_bounds__(PASS_THREADS) tridiag_pass_kernel(double* __restrict__ A, int n, int k, int rows_per,
                                                                    double* __restrict__ scr) {
  __shared__ double s_v[PASS_THREADS], s_w[PASS_THREADS], s_c[PASS_THREADS];
  pdl_launch_dependents();
  pdl_wait();
  const size_t nn = (size_t)n;
  const double* vprev = scr + ((k + 1) & 1) * nn;
  const double* wprev = scr + 2 * nn + ((k + 1) & 1) * nn;
  const double* vcur = scr + (k & 1) * nn;
  double* partial = scr + 4 * nn;
  const int tid = threadIdx.x;
  const int j = k + 1 + blockIdx.x * PASS_THREADS + tid;
  const int r0 = k + 1 + blockIdx.y * rows_per, r1 = min(n, r0 + rows_per);
  const bool col = j < n;
  const double vj = (PREV && col) ? vprev[j] : 0.0, wj = (PREV && col) ? wprev[j] : 0.0;
  double acc = 0.0;
  double* Aj = A + j;
  for (int rb = r0; rb < r1; rb += PASS_THREADS) {
    const int cnt = min(PASS_THREADS, r1 - rb);
    __syncthreads();
    if (tid < cnt) {
      s_c[tid] = vcur[rb + tid];
      if (PREV) { s_v[tid] = vprev[rb + tid]; s_w[tid] = wprev[rb + tid]; }
    }
    __syncthreads();
    if (!col) continue;
    int q = 0;
    for (; q + 8 <= cnt; q += 8) {                     // 8 independent loads in flight before the stores
      double a[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = Aj[(size_t)(rb + q + u) * nn];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (PREV) {
          a[u] = __dsub_rn(a[u], rank2(s_v[q + u], wj, s_w[q + u], vj));
          Aj[(size_t)(rb + q + u) * nn] = a[u];
        }
        acc = fma(a[u], s_c[q + u], acc);
      }
    }
    for (; q < cnt; ++q) {
      double a = Aj[(size_t)(rb + q) * nn];
      if (PREV) {
        a = __dsub_rn(a, rank2(s_v[q], wj, s_w[q], vj));
        Aj[(size_t)(rb + q) * nn] = a;
      }
      acc = fma(a, s_c[q], acc);
    }
  }
  if (col) partial[(size_t)blockIdx.y * nn + j] = acc;
}

// grid of the pass over an m x m trailing block: ~8 CTAs of 256 threads per SM, at most PASS_GY_MAX row tiles
static void pass_grid(int m, int* gx, int* gy, int* rows_per) {
  *gx = (m + PASS_THREADS - 1) / PASS_THREADS;
  int g = (8 * 132 + *gx - 1) / *gx;
  if (g > PASS_GY_MAX) g = PASS_GY_MAX;
  if (g > m) g = m;
  if (g < 1) g = 1;
  *rows_per = (m + g - 1) / g;
  *gy = (m + *rows_per - 1) / *rows_per;
}

// =====================================================================================================================
// (c) Z <- Q Z = H_0 (H_1 (... H_{n-3} Z)), Z [n, kz] row-major, kz <= 16 (dorm2r-style: w = Z' v, Z -= tau v w').
// One cluster of APPLYQ_CTAS CTAs; CTA r keeps rows [r R, (r+1) R) of Z in shared memory (column-major), warp c owns
// column c.  Per reflector: every CTA forms its partial w (one warp-shuffle tree per column), the cluster barrier
// publishes them, and every CTA adds the APPLYQ_CTAS partials in rank order through distributed shared memory.
// =====================================================================================================================
constexpr int APPLYQ_CTAS = 8;
constexpr int APPLYQ_THREADS = 512;

__global__ void __launch_bounds__(APPLYQ_THREADS) apply_q_kernel(const double* __restrict__ A, const double* __restrict__ tau,
                                                                 int n, double* __restrict__ Z, int kz, int R) {
  extern __shared__ double sm[];
  double* part = sm;                                   // [2][16]
  double* vs = sm + 32;                                // [R]
  double* zs = vs + R;                                 // [kz][R]
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int r0 = rank * R, rows = max(0, min(R, n - r0));
  const size_t nn = (size_t)n;
  pdl_launch_dependents();
  pdl_wait();
  for (int q = tid; q < rows * kz; q += APPLYQ_THREADS) {
    const int r = q / kz, c = q - r * kz;
    zs[c * R + r] = Z[(size_t)(r0 + r) * kz + c];
  }
  int par = 0;
  for (int k = n - 3; k >= 0; --k) {
    const double t = tau[k];
    const int lo = max(0, k + 1 - r0);                // first local row with i >= k+1
    for (int r = lo + tid; r < rows; r += APPLYQ_THREADS) {
      const int i = r0 + r;
      vs[r] = i == k + 1 ? 1.0 : A[(size_t)i * nn + k];
    }
    __syncthreads();
    double acc = 0.0;
    if (wid < kz) {
      for (int r = lo + lane; r < rows; r += 32) acc = fma(vs[r], zs[wid * R + r], acc);
      acc = warp_sum_d(acc);
      if (lane == 0) part[par * 16 + wid] = acc;
    }
    cl.sync();
    if (wid < kz) {
      double s = 0.0;
      if (lane < APPLYQ_CTAS) s = cl.map_shared_rank(part, lane)[par * 16 + wid];
      s = warp_sum_d(s);
      const double coef = -t * s;
      for (int r = lo + lane; r < rows; r += 32) zs[wid * R + r] = fma(vs[r], coef, zs[wid * R + r]);
    }
    par ^= 1;
    __syncthreads();
  }
  for (int q = tid; q < rows * kz; q += APPLYQ_THREADS) {
    const int r = q / kz, c = q - r * kz;
    Z[(size_t)(r0 + r) * kz + c] = zs[c * R + r];
  }
  cl.sync();                                           // no CTA leaves while its partials may still be read
}

// ---------------------------------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------------------------------
size_t spectral_scratch_bytes(int n) {
  const size_t nn = (size_t)n;
  const size_t lap = nn * nn * sizeof(float);
  const size_t tri = (4 + PASS_GY_MAX) * nn * sizeof(double);
  return ((lap > tri ? lap : tri) + 255) & ~(size_t)255;
}

int spectral_launches_laplacian() { return 4; }
int spectral_launches_tridiag(int n) { return n >= 2 ? 2 * (n - 2) + 1 : 1; }

static PerDeviceSmem g_prune_smem;

cudaError_t launch_spectral_laplacian(const float* emb, int n, int D, int n_drop, double* L, void* scratch, cudaStream_t st) {
  float* S = reinterpret_cast<float*>(scratch);
  cudaError_t err = launch_cosine_scores(emb, emb, S, n, n, D, st);
  if (err != cudaSuccess) return err;
  const size_t smem = (size_t)n * sizeof(unsigned);
  if (g_prune_smem.need(smem)) {
    err = cudaFuncSetAttribute(prune_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    g_prune_smem.set(smem);
  }
  launch_pdl(prune_rows_kernel, dim3(n), dim3(PRUNE_THREADS), smem, st, S, n, n_drop);
  const int nt = (n + 31) / 32;
  launch_pdl(symmetrize_kernel, dim3(nt, nt), dim3(256), 0, st, (const float*)S, L, n);
  launch_pdl(degree_kernel, dim3(n), dim3(256), 0, st, L, n);
  return cudaGetLastError();
}

cudaError_t launch_sym_tridiag(double* A, int n, double* d, double* e, double* tau, void* scratch, cudaStream_t st) {
  double* scr = reinterpret_cast<double*>(scratch);
  if (n == 1) {
    launch_pdl(reflect_kernel, dim3(1), dim3(REFLECT_THREADS), 0, st, A, n, 0, 0, scr, d, e, tau);
    return cudaGetLastError();
  }
  int gy_prev = 0;
  for (int k = 0; k <= n - 3; ++k) {
    launch_pdl(reflect_kernel, dim3(1), dim3(REFLECT_THREADS), 0, st, A, n, k, gy_prev, scr, d, e, tau);
    int gx, gy, rows_per;
    pass_grid(n - k - 1, &gx, &gy, &rows_per);
    if (k == 0) launch_pdl(tridiag_pass_kernel<false>, dim3(gx, gy), dim3(PASS_THREADS), 0, st, A, n, k, rows_per, scr);
    else launch_pdl(tridiag_pass_kernel<true>, dim3(gx, gy), dim3(PASS_THREADS), 0, st, A, n, k, rows_per, scr);
    gy_prev = gy;
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
  }
  launch_pdl(reflect_kernel, dim3(1), dim3(REFLECT_THREADS), 0, st, A, n, n - 2, gy_prev, scr, d, e, tau);
  return cudaGetLastError();
}

int apply_q_max_rows(int kz) {                         // rows per CTA that fit in shared memory
  return (int)((227 * 1024 / sizeof(double) - 32) / (size_t)(kz + 1));
}

static PerDeviceSmem g_applyq_smem;

cudaError_t launch_sym_tridiag_apply_q(const double* A, const double* tau, int n, double* Z, int kz, cudaStream_t st) {
  if (n < 3) return cudaSuccess;                       // Q = I
  const int R = (n + APPLYQ_CTAS - 1) / APPLYQ_CTAS;
  const size_t smem = (32 + (size_t)R * (kz + 1)) * sizeof(double);
  if (g_applyq_smem.need(smem)) {
    cudaError_t err = cudaFuncSetAttribute(apply_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    g_applyq_smem.set(smem);
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(APPLYQ_CTAS);
  cfg.blockDim = dim3(APPLYQ_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = APPLYQ_CTAS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  return cudaLaunchKernelEx(&cfg, apply_q_kernel, A, tau, n, Z, kz, R);
}

}  // namespace vpb
