// Verification metrics of MVectorTrainer.evaluate (trainer.py:462-468, metric/metrics.py): EER, minDCF and the EER
// threshold of a score list, on the device.
//   (a) stable LSD radix sort of 32-bit order-preserving score keys with a 1-byte label payload: 4 passes of 8 bits, each
//       a per-tile digit histogram (digit-major), a fixed-order exclusive scan over the histograms (reduce, one-CTA top
//       level, down-sweep) and a stable scatter that ranks keys within each digit in index order;
//   (b) curve pass over the sorted labels: per-tile target / impostor counts, the same scan, then at every position
//       fnr = T_i / T, fpr = 1 - I_i / I, gap = fnr - fpr and the detection cost in numpy's operation order, reduced
//       to x1 (first gap >= 0), x2 (last gap < 0), the minimum cost and the first index attaining it.
// No CTA waits on another CTA's flag (reduce-then-scan, no decoupled look-back).  Counts and offsets are integers and
// every floating-point value is formed per position without contraction (__dmul_rn / __dadd_rn / __dsub_rn /
// __ddiv_rn): results are bit-reproducible and equal to the numpy evaluation on the same sorted label sequence.
#include "kernels.cuh"

namespace vpb {

constexpr int VT_THREADS = 256;                  // sort / curve tiles: 256 threads x 16 items
constexpr int VT_ITEMS = 16;
constexpr int VT_TILE = VT_THREADS * VT_ITEMS;   // 4096 scores per tile
constexpr int VT_WARPS = VT_THREADS / 32;
constexpr int SCAN_TOP_THREADS = 1024;

typedef unsigned long long u64;

// Label payload: 1 = target (label == 1), 0 = impostor (label == 0), 2 = neither (counted by neither cumsum, exactly as
// compute_fnr_fpr's `labels == 1` / `labels == 0` weights).
__device__ __forceinline__ uint8_t label_code(int v) { return v == 1 ? 1 : (v == 0 ? 0 : 2); }

// Order-preserving 32-bit key of a score: -0 folds onto +0 (numpy compares them equal), every NaN onto one key above
// +inf (numpy sorts NaNs last).
__device__ __forceinline__ unsigned score_key(float f) {
  if (f != f) return 0xffffffffu;
  const unsigned u = __float_as_uint(f == 0.f ? 0.f : f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct LabelSrc {
  const int32_t* flat;       // [n] or null
  const int32_t* trial;      // matrix form: label of score i is trial[i / n_enroll] == enroll[i % n_enroll]
  const int32_t* enroll;
  unsigned n_enroll;         // n <= 2^31: indices and n_enroll fit in 32 bits here
};

__device__ __forceinline__ uint8_t label_at(const LabelSrc& ls, unsigned i) {
  if (ls.flat) return label_code(ls.flat[i]);
  const unsigned q = i / ls.n_enroll;
  return ls.trial[q] == ls.enroll[i - q * ls.n_enroll] ? 1 : 0;
}

// ---- block-wide exclusive scan of u64 (every thread gets its exclusive prefix and the total) ----
__device__ __forceinline__ u64 warp_incl_u64(u64 v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
__device__ u64 block_excl_u64(u64 v, u64* s /* [33] shared */, u64* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const u64 incl = warp_incl_u64(v, lane);
  __syncthreads();                                     // s may still be read by a previous call
  if (lane == 31) s[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const u64 w = lane < nw ? s[lane] : 0ull;
    const u64 wi = warp_incl_u64(w, lane);
    if (lane < nw) s[lane] = wi - w;
    if (lane == 31) s[32] = wi;
  }
  __syncthreads();
  *total = s[32];
  return s[wid] + incl - v;
}

// =====================================================================================================================
// Exclusive scan of an array of counts in three fixed-order launches: per-chunk sums, one CTA scanning the chunk sums
// (sums[m] = grand total), down-sweep.  T = unsigned (sort histograms: offsets < n <= 2^31) or u64 (packed curve counts).
// =====================================================================================================================
template <typename T>
__global__ void __launch_bounds__(VT_THREADS) scan_reduce_kernel(const T* __restrict__ in, int64_t n, u64* __restrict__ sums) {
  __shared__ u64 s[33];
  pdl_launch_dependents();
  pdl_wait();
  const int64_t base = (int64_t)blockIdx.x * VT_TILE;
  u64 v = 0ull;
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) {
    const int64_t i = base + j * VT_THREADS + threadIdx.x;
    if (i < n) v += in[i];
  }
  u64 tot;
  block_excl_u64(v, s, &tot);
  if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(SCAN_TOP_THREADS) scan_top_kernel(u64* __restrict__ sums, int64_t m) {
  __shared__ u64 s[33];
  pdl_launch_dependents();
  pdl_wait();
  u64 carry = 0ull;
  for (int64_t b = 0; b < m; b += SCAN_TOP_THREADS) {
    const int64_t i = b + threadIdx.x;
    const u64 v = i < m ? sums[i] : 0ull;
    u64 tot;
    const u64 ex = block_excl_u64(v, s, &tot);
    if (i < m) sums[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) sums[m] = carry;
}

template <typename T>
__global__ void __launch_bounds__(VT_THREADS) scan_down_kernel(T* __restrict__ data, int64_t n, const u64* __restrict__ sums) {
  __shared__ u64 s[33];
  pdl_launch_dependents();
  pdl_wait();
  const int64_t base = (int64_t)blockIdx.x * VT_TILE + (int64_t)threadIdx.x * VT_ITEMS;
  T v[VT_ITEMS];
  u64 local = 0ull;
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) {
    v[j] = base + j < n ? data[base + j] : (T)0;
    local += v[j];
  }
  u64 tot;
  u64 run = sums[blockIdx.x] + block_excl_u64(local, s, &tot);
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) {
    if (base + j < n) data[base + j] = (T)run;
    run += v[j];
  }
}

// =====================================================================================================================
// (a) radix sort.  Item r of warp w of tile t is index t*TILE + w*32*ITEMS + r*32 + lane: loads are coalesced and the
// (warp, round, lane) order is the index order, which the stable ranking relies on.
// =====================================================================================================================
template <bool FIRST>
__device__ __forceinline__ unsigned load_key(const float* scores, const unsigned* kin, int64_t i) {
  return FIRST ? score_key(scores[i]) : kin[i];
}

// hist[d * n_tiles + t] = keys of tile t whose digit (key >> shift) & 255 is d
template <bool FIRST>
__global__ void __launch_bounds__(VT_THREADS) radix_hist_kernel(const float* __restrict__ scores, const unsigned* __restrict__ kin,
                                                                int64_t n, int shift, unsigned* __restrict__ hist, int64_t n_tiles) {
  __shared__ unsigned h[VT_WARPS][256];
  pdl_launch_dependents();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int q = tid; q < VT_WARPS * 256; q += VT_THREADS) (&h[0][0])[q] = 0u;
  __syncthreads();
  pdl_wait();
  const int64_t base = (int64_t)blockIdx.x * VT_TILE + wid * 32 * VT_ITEMS + lane;
#pragma unroll 4
  for (int r = 0; r < VT_ITEMS; ++r) {
    const int64_t i = base + r * 32;
    if (i < n) atomicAdd(&h[wid][(load_key<FIRST>(scores, kin, i) >> shift) & 255u], 1u);   // integer: order free
  }
  __syncthreads();
  unsigned c = 0u;
#pragma unroll
  for (int w = 0; w < VT_WARPS; ++w) c += h[w][tid];
  hist[(int64_t)tid * n_tiles + blockIdx.x] = c;
}

// Stable scatter of one tile: rank every key within its digit in index order (warp match + per-warp running counts),
// place the tile digit-sorted in shared memory, then write each digit's run to its scanned global offset with
// consecutive threads on consecutive addresses.  (Min 2 CTAs per SM: without the hint ptxas caps the pass > 0
// instance at 80 registers and spills.)
template <bool FIRST>
__global__ void __launch_bounds__(VT_THREADS, 2) radix_scatter_kernel(const float* __restrict__ scores, LabelSrc ls,
                                                                   const unsigned* __restrict__ kin, const uint8_t* __restrict__ lin,
                                                                   unsigned* __restrict__ kout, uint8_t* __restrict__ lout,
                                                                   int64_t n, int shift, const unsigned* __restrict__ offs,
                                                                   int64_t n_tiles) {
  __shared__ unsigned s_keys[VT_TILE];
  __shared__ uint8_t s_lab[VT_TILE];
  __shared__ unsigned s_wcnt[VT_WARPS][256];
  __shared__ unsigned s_start[256];
  __shared__ unsigned s_goff[256];
  __shared__ u64 s_red[33];
  pdl_launch_dependents();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int q = tid; q < VT_WARPS * 256; q += VT_THREADS) (&s_wcnt[0][0])[q] = 0u;
  pdl_wait();
  s_goff[tid] = offs[(int64_t)tid * n_tiles + blockIdx.x];
  const int64_t tbase = (int64_t)blockIdx.x * VT_TILE;
  const int cnt = (int)min((int64_t)VT_TILE, n - tbase);
  const int wbase = wid * 32 * VT_ITEMS;
  unsigned key[VT_ITEMS], rk[VT_ITEMS];               // rk: rank within (warp, digit) | label << 16
#pragma unroll
  for (int r = 0; r < VT_ITEMS; ++r) {
    const int li = wbase + r * 32 + lane;
    key[r] = 0u;
    rk[r] = 0u;
    if (li < cnt) {
      const int64_t i = tbase + li;
      key[r] = load_key<FIRST>(scores, kin, i);
      rk[r] = (unsigned)(FIRST ? label_at(ls, (unsigned)i) : lin[i]) << 16;
    }
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < VT_ITEMS; ++r) {
    const bool valid = wbase + r * 32 + lane < cnt;
    const unsigned d = valid ? (key[r] >> shift) & 255u : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned before = __popc(peers & lt);
    const unsigned c = valid ? s_wcnt[wid][d] : 0u;
    __syncwarp();
    if (valid && before == 0u) s_wcnt[wid][d] = c + __popc(peers);
    __syncwarp();
    rk[r] |= c + before;
  }
  __syncthreads();
  u64 run = 0ull;                                      // thread tid owns digit tid: exclusive over warps
#pragma unroll
  for (int w = 0; w < VT_WARPS; ++w) {
    const unsigned t = s_wcnt[w][tid];
    s_wcnt[w][tid] = (unsigned)run;
    run += t;
  }
  u64 tot;
  s_start[tid] = (unsigned)block_excl_u64(run, s_red, &tot);
  __syncthreads();
#pragma unroll
  for (int r = 0; r < VT_ITEMS; ++r) {
    if (wbase + r * 32 + lane < cnt) {
      const unsigned d = (key[r] >> shift) & 255u;
      const unsigned pos = s_start[d] + s_wcnt[wid][d] + (rk[r] & 0xffffu);
      s_keys[pos] = key[r];
      s_lab[pos] = (uint8_t)(rk[r] >> 16);
    }
  }
  __syncthreads();
  for (int q = tid; q < cnt; q += VT_THREADS) {
    const unsigned k = s_keys[q];
    const unsigned d = (k >> shift) & 255u;
    const int64_t g = (int64_t)s_goff[d] + (q - (int)s_start[d]);
    kout[g] = k;
    lout[g] = s_lab[q];
  }
}

// =====================================================================================================================
// (b) curve pass over the sorted labels.  Thread tid of tile t owns positions t*TILE + tid*ITEMS + [0, ITEMS).
// Counts are packed as targets + (impostors << 32): both stay below 2^31, so packed sums never carry between halves.
// =====================================================================================================================
struct CurvePartial {
  int64_t x1, x2, arg;       // first gap >= 0 (INT64_MAX: none), last gap < 0 (-1: none), first argmin (INT64_MAX)
  double cost;               // minimum cost (+inf: none)
  u64 c1, c2;                // packed inclusive counts at x1 and x2
};

__device__ __forceinline__ void load_labels(const uint8_t* lab, int64_t p0, int64_t n, uint8_t* out) {
  if (p0 + VT_ITEMS <= n) {
    const uint4 v = *reinterpret_cast<const uint4*>(lab + p0);    // tiles start on 4096-byte offsets of 256-B buffers
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < VT_ITEMS; ++j) out[j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
  } else {
#pragma unroll
    for (int j = 0; j < VT_ITEMS; ++j) out[j] = p0 + j < n ? lab[p0 + j] : (uint8_t)2;
  }
}

__device__ __forceinline__ u64 pack_count(uint8_t c) { return c == 1 ? 1ull : (c == 0 ? (1ull << 32) : 0ull); }

__global__ void __launch_bounds__(VT_THREADS) curve_count_kernel(const uint8_t* __restrict__ lab, int64_t n, u64* __restrict__ tcnt) {
  __shared__ u64 s[33];
  pdl_launch_dependents();
  pdl_wait();
  uint8_t c[VT_ITEMS];
  load_labels(lab, (int64_t)blockIdx.x * VT_TILE + threadIdx.x * VT_ITEMS, n, c);
  u64 v = 0ull;
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) v += pack_count(c[j]);
  u64 tot;
  block_excl_u64(v, s, &tot);
  if (threadIdx.x == 0) tcnt[blockIdx.x] = tot;
}

struct CostParams {
  double p_target, c_miss, c_fa, one_minus_p;    // one_minus_p = 1 - p_target, formed once on the host as numpy does
};

__device__ __forceinline__ void combine(CurvePartial& a, const CurvePartial& b) {
  if (b.x1 < a.x1) { a.x1 = b.x1; a.c1 = b.c1; }
  if (b.x2 > a.x2) { a.x2 = b.x2; a.c2 = b.c2; }
  if (b.cost < a.cost || (b.cost == a.cost && b.arg < a.arg)) { a.cost = b.cost; a.arg = b.arg; }
}

__device__ __forceinline__ CurvePartial shfl_down_partial(const CurvePartial& p, int o) {
  CurvePartial q;
  q.x1 = __shfl_down_sync(0xffffffffu, p.x1, o);
  q.x2 = __shfl_down_sync(0xffffffffu, p.x2, o);
  q.arg = __shfl_down_sync(0xffffffffu, p.arg, o);
  q.cost = __shfl_down_sync(0xffffffffu, p.cost, o);
  q.c1 = __shfl_down_sync(0xffffffffu, p.c1, o);
  q.c2 = __shfl_down_sync(0xffffffffu, p.c2, o);
  return q;
}

__device__ __forceinline__ CurvePartial empty_partial() {
  CurvePartial p;
  p.x1 = INT64_MAX; p.x2 = -1; p.arg = INT64_MAX; p.cost = __longlong_as_double(0x7ff0000000000000ll);
  p.c1 = 0ull; p.c2 = 0ull;
  return p;
}

// The selection is a total order (min index / max index / (cost, index)): the tree's shape cannot change the result.
__device__ CurvePartial block_combine(CurvePartial p, CurvePartial* s /* [32] shared */) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) combine(p, shfl_down_partial(p, o));
  __syncthreads();
  if (lane == 0) s[wid] = p;
  __syncthreads();
  if (wid == 0) {
    p = lane < nw ? s[lane] : empty_partial();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) combine(p, shfl_down_partial(p, o));
  }
  return p;                                            // valid in thread 0
}

__global__ void __launch_bounds__(VT_THREADS) curve_eval_kernel(const uint8_t* __restrict__ lab, const unsigned* __restrict__ keys,
                                                                int64_t n, const u64* __restrict__ toff,
                                                                const u64* __restrict__ total, CostParams cp,
                                                                CurvePartial* __restrict__ part, float* __restrict__ sorted_scores,
                                                                uint8_t* __restrict__ sorted_labels) {
  __shared__ u64 s[33];
  __shared__ CurvePartial s_part[32];
  pdl_launch_dependents();
  pdl_wait();
  const int64_t p0 = (int64_t)blockIdx.x * VT_TILE + threadIdx.x * VT_ITEMS;
  uint8_t c[VT_ITEMS];
  load_labels(lab, p0, n, c);
  u64 local = 0ull;
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) local += pack_count(c[j]);
  u64 tot;
  u64 run = toff[blockIdx.x] + block_excl_u64(local, s, &tot);
  const u64 all = *total;
  const double T = (double)(all & 0xffffffffull), I = (double)(all >> 32);
  CurvePartial best = empty_partial();
#pragma unroll
  for (int j = 0; j < VT_ITEMS; ++j) {
    const int64_t i = p0 + j;
    if (i >= n) continue;
    run += pack_count(c[j]);
    const double fnr = __ddiv_rn((double)(run & 0xffffffffull), T);
    const double fpr = __dsub_rn(1.0, __ddiv_rn((double)(run >> 32), I));
    const double gap = __dsub_rn(fnr, fpr);
    const double cost = __dadd_rn(__dmul_rn(__dmul_rn(cp.c_miss, fnr), cp.p_target),
                                  __dmul_rn(__dmul_rn(cp.c_fa, fpr), cp.one_minus_p));
    if (gap >= 0.0) { if (i < best.x1) { best.x1 = i; best.c1 = run; } }
    else if (gap < 0.0) { best.x2 = i; best.c2 = run; }
    if (cost < best.cost) { best.cost = cost; best.arg = i; }
  }
  if (sorted_scores) {
    for (int j = 0; j < VT_ITEMS; ++j)
      if (p0 + j < n) sorted_scores[p0 + j] = key_score(keys[p0 + j]);
  }
  if (sorted_labels) {
    for (int j = 0; j < VT_ITEMS; ++j)
      if (p0 + j < n) sorted_labels[p0 + j] = c[j];
  }
  best = block_combine(best, s_part);
  if (threadIdx.x == 0) part[blockIdx.x] = best;
}

__global__ void __launch_bounds__(SCAN_TOP_THREADS) curve_final_kernel(const CurvePartial* __restrict__ part, int64_t n_tiles,
                                                                       const u64* __restrict__ total, const unsigned* __restrict__ keys,
                                                                       vp_verify_result* __restrict__ res) {
  __shared__ CurvePartial s_part[32];
  pdl_launch_dependents();
  pdl_wait();
  CurvePartial p = empty_partial();
  for (int64_t t = threadIdx.x; t < n_tiles; t += SCAN_TOP_THREADS) combine(p, part[t]);
  p = block_combine(p, s_part);
  if (threadIdx.x == 0) {
    const u64 all = n_tiles > 0 ? *total : 0ull;
    vp_verify_result r;
    r.n_target = (int64_t)(all & 0xffffffffull);
    r.n_impostor = (int64_t)(all >> 32);
    r.x1 = p.x1 == INT64_MAX ? -1 : p.x1;
    r.x2 = p.x2;
    r.target_x1 = r.x1 >= 0 ? (int64_t)(p.c1 & 0xffffffffull) : 0;
    r.impostor_x1 = r.x1 >= 0 ? (int64_t)(p.c1 >> 32) : 0;
    r.target_x2 = r.x2 >= 0 ? (int64_t)(p.c2 & 0xffffffffull) : 0;
    r.impostor_x2 = r.x2 >= 0 ? (int64_t)(p.c2 >> 32) : 0;
    r.min_cost = p.cost;
    r.argmin = p.arg == INT64_MAX ? -1 : p.arg;
    r.threshold = r.x1 >= 0 ? key_score(keys[r.x1]) : __int_as_float(0x7fffffff);
    r.reserved0 = 0;
    *res = r;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
struct VerifyScratch {
  unsigned* keys[2];
  uint8_t* labs[2];
  unsigned* hist;            // [256][n_tiles]
  u64* ssum;                 // sort-scan chunk sums [ceil(256 n_tiles / TILE) + 1]
  u64* tcnt;                 // [n_tiles] packed counts per curve tile -> exclusive offsets
  u64* csum;                 // curve-scan chunk sums [ceil(n_tiles / TILE) + 1]
  CurvePartial* part;        // [n_tiles]
  size_t bytes;
};

static int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static VerifyScratch verify_layout(int64_t n, char* base) {
  const int64_t nt = cdiv(n, VT_TILE);
  VerifyScratch s;
  size_t off = 0;
  auto take = [&](size_t b) { char* p = base ? base + off : nullptr; off += align256(b); return p; };
  s.keys[0] = reinterpret_cast<unsigned*>(take(4 * (size_t)n));
  s.keys[1] = reinterpret_cast<unsigned*>(take(4 * (size_t)n));
  s.labs[0] = reinterpret_cast<uint8_t*>(take((size_t)n));
  s.labs[1] = reinterpret_cast<uint8_t*>(take((size_t)n));
  s.hist = reinterpret_cast<unsigned*>(take(4 * 256 * (size_t)nt));
  s.ssum = reinterpret_cast<u64*>(take(8 * (size_t)(cdiv(256 * nt, VT_TILE) + 1)));
  s.tcnt = reinterpret_cast<u64*>(take(8 * (size_t)nt));
  s.csum = reinterpret_cast<u64*>(take(8 * (size_t)(cdiv(nt, VT_TILE) + 1)));
  s.part = reinterpret_cast<CurvePartial*>(take(sizeof(CurvePartial) * (size_t)nt));
  s.bytes = off;
  return s;
}

size_t verify_scratch_bytes(int64_t n) { return verify_layout(n, nullptr).bytes; }

template <typename T>
static void launch_scan(T* data, int64_t m, u64* sums, cudaStream_t st) {
  const int64_t chunks = cdiv(m, VT_TILE);
  launch_pdl(scan_reduce_kernel<T>, dim3((unsigned)chunks), dim3(VT_THREADS), 0, st, (const T*)data, m, sums);
  launch_pdl(scan_top_kernel, dim3(1), dim3(SCAN_TOP_THREADS), 0, st, sums, chunks);
  launch_pdl(scan_down_kernel<T>, dim3((unsigned)chunks), dim3(VT_THREADS), 0, st, data, m, (const u64*)sums);
}

cudaError_t launch_verify_sort(const float* scores, const int32_t* labels, const int32_t* trial, const int32_t* enroll,
                               int64_t n_enroll, int64_t n, void* scratch, cudaStream_t st) {
  VerifyScratch s = verify_layout(n, reinterpret_cast<char*>(scratch));
  const int64_t nt = cdiv(n, VT_TILE);
  LabelSrc ls{labels, trial, enroll, (unsigned)(labels ? 1 : n_enroll)};
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 8 * pass;
    const int src = (pass + 1) & 1, dst = pass & 1;    // pass 0: scores -> buffer 0, then 0 -> 1 -> 0 -> 1
    if (pass == 0)
      launch_pdl(radix_hist_kernel<true>, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, scores, (const unsigned*)nullptr, n,
                 shift, s.hist, nt);
    else
      launch_pdl(radix_hist_kernel<false>, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, (const float*)nullptr,
                 (const unsigned*)s.keys[src], n, shift, s.hist, nt);
    launch_scan<unsigned>(s.hist, 256 * nt, s.ssum, st);
    if (pass == 0)
      launch_pdl(radix_scatter_kernel<true>, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, scores, ls,
                 (const unsigned*)nullptr, (const uint8_t*)nullptr, s.keys[dst], s.labs[dst], n, shift,
                 (const unsigned*)s.hist, nt);
    else
      launch_pdl(radix_scatter_kernel<false>, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, (const float*)nullptr, ls,
                 (const unsigned*)s.keys[src], (const uint8_t*)s.labs[src], s.keys[dst], s.labs[dst], n, shift,
                 (const unsigned*)s.hist, nt);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
  }
  return cudaSuccess;
}

cudaError_t launch_verify_curve(int64_t n, double p_target, double c_miss, double c_fa, void* scratch, float* sorted_scores,
                                uint8_t* sorted_labels, vp_verify_result* result, cudaStream_t st) {
  VerifyScratch s = verify_layout(n, reinterpret_cast<char*>(scratch));
  const int64_t nt = cdiv(n, VT_TILE);
  if (nt > 0) {
    launch_pdl(curve_count_kernel, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, (const uint8_t*)s.labs[1], n, s.tcnt);
    launch_scan<u64>(s.tcnt, nt, s.csum, st);
    const CostParams cp{p_target, c_miss, c_fa, 1.0 - p_target};
    launch_pdl(curve_eval_kernel, dim3((unsigned)nt), dim3(VT_THREADS), 0, st, (const uint8_t*)s.labs[1],
               (const unsigned*)s.keys[1], n, (const u64*)s.tcnt, (const u64*)(s.csum + cdiv(nt, VT_TILE)), cp, s.part,
               sorted_scores, sorted_labels);
  }
  launch_pdl(curve_final_kernel, dim3(1), dim3(SCAN_TOP_THREADS), 0, st, (const CurvePartial*)s.part, nt,
             (const u64*)(s.csum + cdiv(nt, VT_TILE)), (const unsigned*)s.keys[1], result);
  return cudaGetLastError();
}

}  // namespace vpb
