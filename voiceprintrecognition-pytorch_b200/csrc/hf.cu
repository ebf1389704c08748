// Hugging Face wav2vec 2.0 / WavLM front-end (include/vpb200.h, vp_frontend_set_hf): the processor's row normalisation,
// the convolutional feature encoder and the feature projection's LayerNorm, then CMN and the keep mask.
//
//   hf_normalize_kernel   one CTA per row: numpy's float32 mean / var of Wav2Vec2FeatureExtractor bit for bit, writing
//                         the normalised row as [rows of s_0 samples, padded to cp channels] -- the layout that makes
//                         layer 0 (k_0 = kt_0 s_0) a kt_0-tap, stride-1 conv with cp input channels.
//   conv layers           the split-TF32 tensor-core engine (launch_conv_tc), GELU fused into its epilogue where no norm
//                         sits between the conv and the activation.  Split TF32 has no call-wide activation scale, so an
//                         output row depends on its own receptive field only: rows are independent of each other and of
//                         how a call is sliced.
//   hf_groupnorm_kernel   "group" layer 0: per (row, channel) mean / biased variance over the row's own frames (fp64),
//                         affine, GELU, in place.
//   hf_layernorm_kernel   one warp per frame: LayerNorm over the channels (+ GELU), in place.
//   hf_cmn_kernel         per (row, channel) mean over the row's frames, subtracted, frames past keep zeroed -> feats.
// A call runs over slices of rows whose scratch stays below VP_HF_SCRATCH_CAP floats.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.cuh"

namespace vpb {

struct HfLayer {
  int cin, cout, k, s;      // as configured (layer 0: cin = 1)
  int kt, cp;               // as run: taps and input channels (layer 0: k / s taps over rows of s samples padded to cp)
  int bn, kc;               // N tile of the tensor-core image, accumulation chunk (vp_op.tc_kc)
  float* w_tc = nullptr;    // pack_tc image of the [cout, kt * cp] weight
  float* bias = nullptr;
  float* g = nullptr;       // norm affine (layer 0 of "group", every layer of "layer")
  float* b = nullptr;
};

struct HfState {
  vp_hf_desc d;
  HfLayer L[VP_HF_MAX_LAYERS];
  float* proj_g = nullptr;
  float* proj_b = nullptr;
  int cmax = 0;
};

namespace {

constexpr int NORM_THREADS = 256;
constexpr int NORM_DEPTH = 8;                  // 2^8 = NORM_THREADS subtrees of the pairwise tree per row
constexpr int LN_WARPS = 8;
constexpr int LN_MAX_VEC = 8;                  // float4 per lane: C <= 1024

__device__ __forceinline__ float gelu(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }

// ---- numpy's float32 pairwise sum (umath loops_utils.h, PW_BLOCKSIZE 128), optionally of the squares of (a - mean) ----
template <bool SQ>
__device__ __forceinline__ float pw_load(const float* a, int64_t i, float mean) {
  float v = a[i];
  if (SQ) {
    v = __fsub_rn(v, mean);
    v = __fmul_rn(v, v);
  }
  return v;
}

template <bool SQ>
__device__ float pw_leaf(const float* a, int64_t n, float mean) {
  if (n < 8) {
    float r = 0.f;
    for (int64_t i = 0; i < n; ++i) r = __fadd_rn(r, pw_load<SQ>(a, i, mean));
    return r;
  }
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = pw_load<SQ>(a, j, mean);
  int64_t i = 8;
  for (; i < n - n % 8; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], pw_load<SQ>(a, i + j, mean));
  }
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __fadd_rn(res, pw_load<SQ>(a, i, mean));
  return res;
}

__device__ __forceinline__ int64_t pw_split(int64_t n) {
  const int64_t n2 = n / 2;
  return n2 - n2 % 8;
}

// a whole subtree, serially: post-order walk with an explicit stack (depth < 40 for any int64 length)
template <bool SQ>
__device__ float pw_serial(const float* a, int64_t n, float mean) {
  float left[40];
  int64_t off = 0, len = n;
  int depth = 0;
  uint64_t rbits = 0;                       // bit d: the node at depth d + 1 of the current path is a right child
  int64_t lens_[40];                        // length of the parent at each depth (to find the right sibling)
  int64_t offs_[40];
  float s;
  for (;;) {
    while (len > 128) {
      lens_[depth] = len;
      offs_[depth] = off;
      len = pw_split(len);
      rbits &= ~(1ull << depth);
      ++depth;
    }
    s = pw_leaf<SQ>(a + off, len, mean);
    while (depth > 0 && ((rbits >> (depth - 1)) & 1ull)) {      // a right child: its parent is complete
      --depth;
      s = __fadd_rn(left[depth], s);
    }
    if (depth == 0) return s;
    left[depth - 1] = s;                                          // a left child: descend into its right sibling
    rbits |= 1ull << (depth - 1);
    const int64_t pl = lens_[depth - 1], h = pw_split(pl);
    off = offs_[depth - 1] + h;
    len = pl - h;
  }
}

// The whole row's pairwise sum with NORM_THREADS threads: thread t takes the subtree at depth NORM_DEPTH whose path is
// the bits of t (nothing when the path ends in a leaf above that depth and t's remaining bits are not all 0), then the
// top NORM_DEPTH levels are combined in the tree's own order.  Every thread of the CTA must call; all get the sum.
template <bool SQ>
__device__ float pw_row(const float* a, int64_t n, float mean, float* red) {
  const int t = threadIdx.x;
  int64_t off = 0, len = n;
  bool own = true;
  for (int lv = 0; lv < NORM_DEPTH; ++lv) {
    const int bit = (t >> (NORM_DEPTH - 1 - lv)) & 1;
    if (len > 128) {
      const int64_t h = pw_split(len);
      if (bit) { off += h; len -= h; } else { len = h; }
    } else if (bit) {
      own = false;
    }
  }
  red[t] = own ? pw_serial<SQ>(a + off, len, mean) : 0.f;
  __syncthreads();
  for (int lv = NORM_DEPTH - 1; lv >= 0; --lv) {                  // nodes at depth lv combine their two children
    const int span = 1 << (NORM_DEPTH - lv);
    if (t < (1 << lv)) {
      int64_t l2 = n;                                             // this node's length: walk down from the root
      for (int j = 0; j < lv; ++j) {
        if (l2 <= 128) break;
        const int64_t h = pw_split(l2);
        l2 = ((t >> (lv - 1 - j)) & 1) ? l2 - h : h;
      }
      if (l2 > 128) red[t * span] = __fadd_rn(red[t * span], red[t * span + span / 2]);
    }
    __syncthreads();
  }
  const float s = red[0];
  __syncthreads();
  return __fadd_rn(0.f, s);                                       // the reduction starts from add's identity
}

__global__ void __launch_bounds__(NORM_THREADS) hf_normalize_kernel(const float* __restrict__ wave, int64_t ld, int L,
                                                                    const int* __restrict__ lens, int do_norm, int s0,
                                                                    int cp, int rows, float* __restrict__ x0) {
  __shared__ float red[NORM_THREADS];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const float* a = wave + (int64_t)b * ld;
  const int64_t n = lens ? (int64_t)lens[b] : (int64_t)L;
  float mean = 0.f, denom = 1.f;
  if (do_norm && n > 0) {
    // x.mean(): float32 pairwise sum, divided by the intp count in float64 and rounded to float32 (numpy _mean)
    mean = (float)((double)pw_row<false>(a, n, 0.f, red) / (double)n);
    const float var = (float)((double)pw_row<true>(a, n, mean, red) / (double)n);
    denom = __fsqrt_rn(__fadd_rn(var, 1e-7f));
  }
  float* out = x0 + (int64_t)b * rows * cp;
  for (int64_t i = threadIdx.x; i < (int64_t)rows * cp; i += NORM_THREADS) {
    const int64_t r = i / cp;
    const int c = (int)(i - r * cp);
    const int64_t j = r * s0 + c;
    float v = 0.f;
    if (c < s0 && j < n) {
      v = a[j];
      if (do_norm) v = __fdiv_rn(__fsub_rn(v, mean), denom);
    }
    out[i] = v;
  }
}

__host__ __device__ inline int conv_frames(int64_t n, int k, int s) { return n < k ? 0 : (int)((n - k) / s + 1); }

struct Geo {          // frame geometry, device-visible copy of the layer kernels / strides
  int n, k[VP_HF_MAX_LAYERS], s[VP_HF_MAX_LAYERS];
};
__host__ __device__ inline int geo_frames(const Geo& g, int64_t n, int upto) {   // frames after layers 0 .. upto
  int64_t t = n;
  for (int l = 0; l <= upto; ++l) t = conv_frames(t, g.k[l], g.s[l]);
  return (int)t;
}

// GroupNorm(C groups) of layer 0 + GELU, in place over x [B, T0, C]: stats over the row's own T_b frames
__global__ void __launch_bounds__(256) hf_groupnorm_kernel(float* __restrict__ x, int T0, int C,
                                                           const int* __restrict__ lens, Geo geo, const float* __restrict__ g,
                                                           const float* __restrict__ bta, float eps) {
  __shared__ double red[8][33];
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x, b = blockIdx.y, ty = threadIdx.y;
  const int Tb = lens ? geo_frames(geo, lens[b], 0) : T0;
  float* row = x + (int64_t)b * T0 * C;
  const bool on = c < C;
  double s = 0.0;
  if (on) for (int t = ty; t < Tb; t += 8) s += (double)row[(int64_t)t * C + c];
  red[ty][threadIdx.x] = s;
  __syncthreads();
  double tot = 0.0;
  for (int j = 0; j < 8; ++j) tot += red[j][threadIdx.x];
  const double mean = Tb > 0 ? tot / Tb : 0.0;
  __syncthreads();
  s = 0.0;
  if (on) for (int t = ty; t < Tb; t += 8) { const double d = (double)row[(int64_t)t * C + c] - mean; s += d * d; }
  red[ty][threadIdx.x] = s;
  __syncthreads();
  tot = 0.0;
  for (int j = 0; j < 8; ++j) tot += red[j][threadIdx.x];
  if (!on) return;
  const double rstd = 1.0 / sqrt((Tb > 0 ? tot / Tb : 0.0) + (double)eps);
  const float sc = (float)rstd * g[c], sh = bta[c] - (float)(mean * rstd) * g[c];
  for (int t = ty; t < T0; t += 8) {
    float& v = row[(int64_t)t * C + c];
    v = gelu(fmaf(v, sc, sh));
  }
}

// LayerNorm over the C channels of each of `rows` rows (+ GELU), one warp per row, in place
__global__ void __launch_bounds__(LN_WARPS * 32) hf_layernorm_kernel(float* __restrict__ x, int64_t rows, int C,
                                                                     const float* __restrict__ g,
                                                                     const float* __restrict__ bta, float eps, int act) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (r >= rows) return;
  float4* p = reinterpret_cast<float4*>(x + r * C);
  const int nv = C >> 2;
  float4 v[LN_MAX_VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < nv ? p[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    if (lane + 32 * i < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = 1.f / sqrtf(warp_sum(q) / (float)C + eps);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(bta);
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) {
      const float4 gg = g4[j], bb = b4[j];
      float4 o;
      o.x = fmaf((v[i].x - mean) * rstd, gg.x, bb.x);
      o.y = fmaf((v[i].y - mean) * rstd, gg.y, bb.y);
      o.z = fmaf((v[i].z - mean) * rstd, gg.z, bb.z);
      o.w = fmaf((v[i].w - mean) * rstd, gg.w, bb.w);
      if (act) { o.x = gelu(o.x); o.y = gelu(o.y); o.z = gelu(o.z); o.w = gelu(o.w); }
      p[j] = o;
    }
  }
}

// CMN over the row's own frames + keep mask: x [B, Tx, C] -> feats [B, T, C]
__global__ void __launch_bounds__(256) hf_cmn_kernel(const float* __restrict__ x, int Tx, int C, float* __restrict__ feats,
                                                     int T, const int* __restrict__ lens, Geo geo,
                                                     const int* __restrict__ keep) {
  __shared__ double red[8][33];
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x, b = blockIdx.y, ty = threadIdx.y;
  const int Tb = lens ? geo_frames(geo, lens[b], geo.n - 1) : T;
  const int kb = keep ? min(keep[b], Tb) : Tb;
  const float* row = x + (int64_t)b * Tx * C;
  const bool on = c < C;
  double s = 0.0;
  if (on) for (int t = ty; t < Tb; t += 8) s += (double)row[(int64_t)t * C + c];
  red[ty][threadIdx.x] = s;
  __syncthreads();
  double tot = 0.0;
  for (int j = 0; j < 8; ++j) tot += red[j][threadIdx.x];
  if (!on) return;
  const float mean = Tb > 0 ? (float)(tot / Tb) : 0.f;
  float* out = feats + (int64_t)b * T * C;
  for (int t = ty; t < T; t += 8) out[(int64_t)t * C + c] = t < kb ? row[(int64_t)t * C + c] - mean : 0.f;
}

// mvector/engine.py::pack_tc: [N, K] -> split-TF32 image [n_tiles][k_blocks][hi|lo][bn][32], 16-byte chunks swizzled
std::vector<float> pack_tc_image(const std::vector<float>& W, int N, int K, int bn) {
  const int nt = (N + bn - 1) / bn, kb = (K + 31) / 32;
  std::vector<float> out((size_t)nt * kb * 2 * bn * 32, 0.f);
  for (int n = 0; n < nt * bn; ++n)
    for (int k = 0; k < kb * 32; ++k) {
      const float w = (n < N && k < K) ? W[(size_t)n * K + k] : 0.f;
      uint32_t u;
      memcpy(&u, &w, 4);
      u = (u + 0x1000u) & 0xFFFFE000u;                               // cvt.rna.tf32.f32
      float hi;
      memcpy(&hi, &u, 4);
      const float lo = w - hi;
      const int tile = n / bn, r = n % bn, kbi = k / 32, c = (k % 32) / 4, e = k % 4;
      for (int p = 0; p < 2; ++p) {
        const size_t idx = (((((size_t)tile * kb + kbi) * 2 + p) * bn + r) * 8 + (c ^ (r & 7))) * 4 + e;
        out[idx] = p == 0 ? hi : lo;
      }
    }
  return out;
}

int tile_n(int N, bool chunked) {
  const int cap = chunked ? 64 : 128;
  return N >= cap ? cap : (N + 15) / 16 * 16;
}

size_t al64(size_t n) { return (n + 63) & ~(size_t)63; }

Geo geo_of(const HfState* s) {
  Geo g{};
  g.n = s->d.n_layers;
  for (int l = 0; l < g.n; ++l) { g.k[l] = s->d.conv_kernel[l]; g.s[l] = s->d.conv_stride[l]; }
  return g;
}

// the largest layer-0 frame count whose stack yields T output frames
int t0_bound(const HfState* s, int T) {
  int64_t t = T;
  for (int l = s->d.n_layers - 1; l >= 1; --l) t = (t - 1) * s->d.conv_stride[l] + s->d.conv_kernel[l] + s->d.conv_stride[l] - 1;
  return (int)(t < (1 << 30) ? t : (1 << 30));
}

size_t row_floats(const HfState* s, int T0) {
  const HfLayer& l0 = s->L[0];
  return al64((size_t)(T0 + l0.kt - 1) * l0.cp) + 2 * al64((size_t)T0 * s->cmax);
}

int slice_rows(const HfState* s, int B, int T0) {
  const size_t per = row_floats(s, T0);
  size_t S = per > 0 ? VP_HF_SCRATCH_CAP / per : (size_t)B;
  if (S < 1) S = 1;
  return S < (size_t)B ? (int)S : B;
}

template <typename T>
cudaError_t upload(T** dst, const T* src, size_t n) {
  cudaError_t e = cudaMalloc(dst, sizeof(T) * (n > 0 ? n : 1));
  if (e != cudaSuccess) return e;
  return cudaMemcpy(*dst, src, sizeof(T) * n, cudaMemcpyHostToDevice);
}

}  // namespace

const char* hf_desc_error(const vp_hf_desc& d) {
  if (d.n_layers < 1 || d.n_layers > VP_HF_MAX_LAYERS) return "n_layers must be in [1, 8]";
  if (d.norm != VP_HF_NORM_GROUP && d.norm != VP_HF_NORM_LAYER) return "norm must be VP_HF_NORM_GROUP or _LAYER";
  for (int l = 0; l < d.n_layers; ++l) {
    if (d.conv_dim[l] < 16 || d.conv_dim[l] > 1024 || (d.conv_dim[l] & 3)) return "conv_dim: multiples of 4 in [16, 1024]";
    if (d.conv_kernel[l] < 1 || d.conv_stride[l] < 1) return "conv_kernel / conv_stride must be >= 1";
  }
  if (d.conv_stride[0] > 16 || d.conv_kernel[0] % d.conv_stride[0])
    return "layer 0 needs conv_kernel a multiple of conv_stride, conv_stride <= 16";
  if (!(d.norm_eps > 0.f) || !(d.proj_eps > 0.f)) return "norm_eps / proj_eps must be > 0";
  return "";
}

void hf_destroy(HfState* s) {
  if (!s) return;
  for (auto& l : s->L) { cudaFree(l.w_tc); cudaFree(l.bias); cudaFree(l.g); cudaFree(l.b); }
  cudaFree(s->proj_g);
  cudaFree(s->proj_b);
  delete s;
}

cudaError_t hf_create(const vp_hf_desc& d, const float* const* conv_w, const float* const* conv_b,
                      const float* const* norm_w, const float* const* norm_b, const float* proj_w, const float* proj_b,
                      HfState** out) {
  HfState* s = new HfState();
  s->d = d;
  cudaError_t e = cudaSuccess;
  for (int l = 0; l < d.n_layers && e == cudaSuccess; ++l) {
    HfLayer& L = s->L[l];
    L.cin = l == 0 ? 1 : d.conv_dim[l - 1];
    L.cout = d.conv_dim[l];
    L.k = d.conv_kernel[l];
    L.s = d.conv_stride[l];
    L.kt = l == 0 ? L.k / L.s : L.k;
    L.cp = l == 0 ? (L.s + 3) / 4 * 4 : L.cin;
    const int K = L.kt * L.cp;
    // the tensor core truncates on every accumulate: the long-K layers (K = 1536 / 1024 at the base geometry) sum
    // 256-element chunks in fp32 instead, which keeps the stack within 1e-4 of the fp64 value of its formula
    L.kc = K > 512 ? 256 : 0;
    L.bn = tile_n(L.cout, L.kc > 0);
    if (L.cout > s->cmax) s->cmax = L.cout;
    std::vector<float> W((size_t)L.cout * K, 0.f);      // element (n, kt * cp + ci), channel-last taps
    for (int n = 0; n < L.cout; ++n)
      for (int kt = 0; kt < L.kt; ++kt)
        for (int ci = 0; ci < L.cp; ++ci) {
          float w = 0.f;
          if (l == 0) { if (ci < L.s) w = conv_w[l][(size_t)n * L.k + kt * L.s + ci]; }
          else w = conv_w[l][((size_t)n * L.cin + ci) * L.k + kt];
          W[(size_t)n * K + kt * L.cp + ci] = w;
        }
    const std::vector<float> img = pack_tc_image(W, L.cout, K, L.bn);
    e = upload(&L.w_tc, img.data(), img.size());
    if (e == cudaSuccess && d.conv_bias) e = upload(&L.bias, conv_b[l], (size_t)L.cout);
    if (e == cudaSuccess && (d.norm == VP_HF_NORM_LAYER || l == 0)) {
      e = upload(&L.g, norm_w[l], (size_t)L.cout);
      if (e == cudaSuccess) e = upload(&L.b, norm_b[l], (size_t)L.cout);
    }
  }
  const int F = d.conv_dim[d.n_layers - 1];
  if (e == cudaSuccess) e = upload(&s->proj_g, proj_w, (size_t)F);
  if (e == cudaSuccess) e = upload(&s->proj_b, proj_b, (size_t)F);
  if (e != cudaSuccess) { hf_destroy(s); return e; }
  *out = s;
  return cudaSuccess;
}

int hf_frames(const HfState* s, int64_t n) { return geo_frames(geo_of(s), n, s->d.n_layers - 1); }
int hf_feature_dim(const HfState* s) { return s->d.conv_dim[s->d.n_layers - 1]; }
int hf_min_samples(const HfState* s) {
  int64_t t = 1;
  for (int l = s->d.n_layers - 1; l >= 0; --l) t = (t - 1) * s->d.conv_stride[l] + s->d.conv_kernel[l];
  return (int)t;
}

size_t hf_scratch_floats(const HfState* s, int B, int L) {
  const int T = hf_frames(s, L);
  if (T < 1 || B < 1) return 0;
  const int T0 = t0_bound(s, T);
  return (size_t)slice_rows(s, B, T0) * row_floats(s, T0);
}

void hf_plan(const HfState* s, int B, int L, int32_t* info) {
  const int T = hf_frames(s, L), T0 = conv_frames(L, s->d.conv_kernel[0], s->d.conv_stride[0]);
  const int S = slice_rows(s, B, t0_bound(s, T));
  info[0] = S; info[1] = (B + S - 1) / S; info[2] = T0; info[3] = s->d.n_layers; info[4] = T;
  info[5] = s->L[0].kt; info[6] = s->L[0].cp; info[7] = 0;
}

cudaError_t hf_run(const HfState* s, const float* wave, int B, int ld, const int* lens, int T, const int* keep, float* feats,
                   float* scratch, cudaStream_t st) {
  const vp_hf_desc& d = s->d;
  const Geo geo = geo_of(s);
  const int nl = d.n_layers, F = hf_feature_dim(s);
  const int T0b = t0_bound(s, T);
  int Tl[VP_HF_MAX_LAYERS];
  Tl[0] = conv_frames(ld, d.conv_kernel[0], d.conv_stride[0]);
  if (lens && Tl[0] > T0b) Tl[0] = T0b;            // a ragged call runs the frames of its longest row at most
  for (int l = 1; l < nl; ++l) Tl[l] = conv_frames(Tl[l - 1], d.conv_kernel[l], d.conv_stride[l]);
  const HfLayer& l0 = s->L[0];
  const int R0 = Tl[0] + l0.kt - 1;
  const int S = slice_rows(s, B, T0b);
  for (int b0 = 0; b0 < B; b0 += S) {
    const int n = B - b0 < S ? B - b0 : S;
    // slice scratch: [S rows of the normalised waveform] [S rows of layer output] x 2 (ping-pong)
    float* x0 = scratch;
    float* buf[2];
    buf[0] = x0 + (size_t)S * al64((size_t)R0 * l0.cp);
    buf[1] = buf[0] + (size_t)S * al64((size_t)Tl[0] * s->cmax);
    const int* ln = lens ? lens + b0 : nullptr;
    launch_pdl(hf_normalize_kernel, dim3(n), dim3(NORM_THREADS), 0, st, wave + (int64_t)b0 * ld, (int64_t)ld, ld, ln,
               d.do_normalize, l0.s, l0.cp, R0, x0);
    for (int l = 0; l < nl; ++l) {
      const HfLayer& L = s->L[l];
      ConvParams c{};
      c.src = l == 0 ? x0 : buf[(l - 1) & 1];
      c.dst = buf[l & 1];
      c.w_tc = L.w_tc; c.tc_bn = L.bn; c.tc_kc = L.kc; c.bias = L.bias;
      c.B = n; c.Tin = l == 0 ? R0 : Tl[l - 1]; c.Fin = 1; c.Cin = L.cp; c.CinTot = L.cp; c.in_ld = L.cp;
      c.Tout = Tl[l]; c.Fout = 1; c.out_ld = L.cout;
      c.KT = L.kt; c.KF = 1; c.sT = l == 0 ? 1 : L.s; c.sF = 1; c.dT = 1; c.dF = 1; c.pad_mode = VP_PAD_ZERO;
      c.w_ld = L.kt * L.cp;
      const bool norm_here = d.norm == VP_HF_NORM_LAYER || l == 0;
      c.act = norm_here ? VP_ACT_NONE : VP_ACT_GELU;
      c.act2 = VP_ACT_NONE;
      c.seg_len = 1; c.n_seg = 1;
      c.M = n * Tl[l]; c.N = L.cout; c.K = L.kt * L.cp;
      cudaError_t e = launch_conv_tc(c, st);
      if (e != cudaSuccess) return e;
      if (d.norm == VP_HF_NORM_GROUP && l == 0) {
        launch_pdl(hf_groupnorm_kernel, dim3((L.cout + 31) / 32, n), dim3(32, 8), 0, st, buf[0], Tl[0], L.cout, ln, geo,
                   (const float*)L.g, (const float*)L.b, d.norm_eps);
      } else if (d.norm == VP_HF_NORM_LAYER) {
        const int64_t rows = (int64_t)n * Tl[l];
        launch_pdl(hf_layernorm_kernel, dim3((unsigned)((rows + LN_WARPS - 1) / LN_WARPS)), dim3(LN_WARPS * 32), 0, st,
                   buf[l & 1], rows, L.cout, (const float*)L.g, (const float*)L.b, d.norm_eps, 1);
      }
    }
    float* last = buf[(nl - 1) & 1];
    const int64_t rows = (int64_t)n * Tl[nl - 1];
    launch_pdl(hf_layernorm_kernel, dim3((unsigned)((rows + LN_WARPS - 1) / LN_WARPS)), dim3(LN_WARPS * 32), 0, st, last,
               rows, F, (const float*)s->proj_g, (const float*)s->proj_b, d.proj_eps, 0);
    launch_pdl(hf_cmn_kernel, dim3((F + 31) / 32, n), dim3(32, 8), 0, st, (const float*)last, Tl[nl - 1], F,
               feats + (int64_t)b0 * T * F, T, ln, geo, keep ? keep + b0 : nullptr);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace vpb
