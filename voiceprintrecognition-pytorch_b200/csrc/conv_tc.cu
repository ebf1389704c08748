// Tensor-core engine: implicit-GEMM convolution on the Hopper tensor cores (wgmma) with fp32-grade accuracy
// (split TF32, "3xTF32").
//
//   out[m, n] = epi( sum_k A(m, k) * W[n, k] )        same op contract as conv_ffma.cu (common.cuh::ConvParams)
//
// Why split TF32: a single TF32 (or BF16) pass breaks the 1e-4 embedding parity gate (SURVEY.md 9.3: 3e-4 / 2.7e-3),
// so every operand is split  x = hi + lo,  hi = tf32(x),  lo = x - hi  and three MMAs are accumulated in fp32:
//   D += A_lo * B_hi;  D += A_hi * B_lo;  D += A_hi * B_hi        (the dropped lo*lo term is ~2^-22 relative).
//
// Persistent, warp-specialised CTA (512 threads: 128 registers each), one CTA per SM, 128 x BN output tiles:
//   warps 0-7  consumers  : two warpgroups, each owning 64 rows of the tile, issue wgmma.m64nBNk8 (tf32) from the
//                           shared-memory stage into register accumulators, then run the fused epilogue (bias / ubias /
//                           act / BN affine / gate / residual / act2) straight from the accumulator fragments: every
//                           float2 store of a quad of lanes covers one whole 32-byte sector of an output row
//   warps 8-15 A producers: gather the implicit-GEMM A tile straight from the channel-last activation map (any tap /
//                           dilation / stride / reflect or zero padding / add or concat second source / BN-ReLU
//                           prologue: common.cuh::gather_a4) with coalesced 128 B row segments, split into hi / lo and
//                           write both in the K-major SWIZZLE_128B shared-memory layout the wgmma descriptors read;
//                           weights are pre-split and pre-tiled on the host in exactly that shared-memory image, so one
//                           bulk-async copy (TMA engine, cp.async.bulk) per stage, issued by producer thread 0 as soon
//                           as the stage is free, lands B_hi|B_lo
// Pipeline: S shared-memory stages (full/empty mbarriers); a stage is released as soon as the wgmma group that read
// it has retired, while the next K block's group is already in flight.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>

#include <cstdlib>
#include <type_traits>

#include "kernels.cuh"
#include "wgmma.cuh"

namespace vpb {

namespace tc {

constexpr int BM = 128;
constexpr int BK = 32;                  // fp32 elements per stage row = 128 B = one SWIZZLE_128B row
constexpr int A_TILE = BM * BK * 4;     // 16 KB per (hi|lo) A tile
constexpr int CONSUMER_WARPS = 8;       // two warpgroups x 64 rows
constexpr int CONSUMER_THREADS = CONSUMER_WARPS * 32;
constexpr int PRODUCER_WARPS = 8;
constexpr int PRODUCER_THREADS = PRODUCER_WARPS * 32;      // 256
constexpr int NUM_THREADS = CONSUMER_THREADS + PRODUCER_THREADS;
constexpr int ROWS_PER_THREAD = BM * 8 / PRODUCER_THREADS;   // 4
constexpr int MAX_BN = 128;             // 64 accumulator registers per consumer thread
constexpr int MAX_BN_CHUNKED = 64;      // chunked accumulation keeps a second (running-sum) register set
constexpr int SMEM_BUDGET = 225 * 1024; // pipeline stages (+ 1 KB alignment, + static barriers <= 227 KB)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across wgmma issue / wait
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA): start>>4 | LBO = 16 B (unused when swizzled) |
// SBO = 1024 B (8 rows x 128 B) | layout type 1 (SWIZZLE_128B) at bits 62-63
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr) {
  return (uint64_t)((addr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// D[64 x BN] (+)= A[64 x 8|16] * B[BN x 8|16]^T for one warpgroup.  BN is a multiple of 16 up to 128: it is issued as
// n128, or as n64 / n32 / n16 pieces (B rows of a piece start at a multiple of 16 rows = 2 KB: swizzle atoms stay aligned).
template <int BN, bool F16>
__device__ __forceinline__ void mma_tile(float* d, uint32_t a, uint32_t b, uint32_t scale_d) {
  const uint64_t da = smem_desc(a);
  if constexpr (BN == 128) {
    if constexpr (F16) wgmma_f16_n128(d, da, smem_desc(b), scale_d);
    else wgmma_tf32_n128(d, da, smem_desc(b), scale_d);
  } else {
    constexpr int o64 = 0, o32 = o64 + (BN & 64), o16 = o32 + (BN & 32);
    if constexpr ((BN & 64) != 0) {
      if constexpr (F16) wgmma_f16_n64(d + o64 / 2, da, smem_desc(b + o64 * 128), scale_d);
      else wgmma_tf32_n64(d + o64 / 2, da, smem_desc(b + o64 * 128), scale_d);
    }
    if constexpr ((BN & 32) != 0) {
      if constexpr (F16) wgmma_f16_n32(d + o32 / 2, da, smem_desc(b + o32 * 128), scale_d);
      else wgmma_tf32_n32(d + o32 / 2, da, smem_desc(b + o32 * 128), scale_d);
    }
    if constexpr ((BN & 16) != 0) {
      if constexpr (F16) wgmma_f16_n16(d + o16 / 2, da, smem_desc(b + o16 * 128), scale_d);
      else wgmma_tf32_n16(d + o16 / 2, da, smem_desc(b + o16 * 128), scale_d);
    }
  }
}

__device__ __noinline__ float2 act2_slow(float2 v, int act) {
  v.x = apply_act(v.x, act); v.y = apply_act(v.y, act);
  return v;
}

// Per-launch epilogue flags.  ReLU and the ERes2Net family's ReLU(20) = Hardtanh(0, 20) (eres2net.py:12-17) are both
// "clamp to [0, hi]" with hi = +inf / 20: min(max(x, 0), hi), the same expression and order as apply_act.
struct Epi {
  bool simple, relu, relu2, need_urow;
  float hi1, hi2;
  float descale;         // fp16 split: 2^-k of the weight image x 2^-s of the activation scale; 1 on the tf32 path
};
__device__ __forceinline__ Epi make_epi(const ConvParams& p, float descale) {
  auto clamps = [](int act) { return act == VP_ACT_RELU || act == VP_ACT_HARDTANH20; };
  Epi e;
  e.simple = !p.ubias && !p.gate && !p.sum && (p.act == VP_ACT_NONE || clamps(p.act)) &&
             (p.act2 == VP_ACT_NONE || clamps(p.act2));
  e.relu = clamps(p.act);
  e.relu2 = clamps(p.act2);
  e.hi1 = p.act == VP_ACT_HARDTANH20 ? 20.f : INFINITY;
  e.hi2 = p.act2 == VP_ACT_HARDTANH20 ? 20.f : INFINITY;
  e.need_urow = (p.gate != nullptr) || (p.ubias != nullptr);
  e.descale = descale;
  return e;
}

// Residual tiles are pure streaming: pull tile gg's residual rows (this consumer warp's 16) into the L2 while the
// current tile's MMAs run, so that the epilogue's residual loads are L2 hits.
template <int BN>
__device__ __forceinline__ void prefetch_res(const ConvParams& p, int gg, int n_tiles, int warp, int lane) {
  if (!p.res) return;
  const int mr = (gg / n_tiles) * BM + 64 * (warp >> 2) + 16 * (warp & 3) + (lane & 15);
  const float* base = p.res + p.res_coff + (gg % n_tiles) * BN;
  if (mr < p.M)
    for (int c = 32 * (lane >> 4); c < BN; c += 64)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(base + (size_t)mr * p.res_ld + c));
}

// Fused epilogue of one consumer thread's share of a BM x BN tile, straight from the wgmma accumulator fragments
// (res[4j + 2h + c] = row ma + 8h, column n0 + 8j + 2 q4 + c): every float2 store of a quad of lanes covers one whole
// 32-byte sector of an output row.  tmax collects max |y| of what is stored (amax_out slot).
template <int BN>
__device__ __forceinline__ void store_tile(const ConvParams& p, const Epi& e, const float (&res)[BN / 2], int m0, int n0,
                                           int ma, int q4, float& tmax) {
  const float descale = e.descale;
  if (e.simple && m0 + BM <= p.M && n0 + BN <= p.N) {
    // Fast path: the common epilogue shape -- bias, optional ReLU, optional BN affine, optional residual, nothing
    // per utterance -- on a tile without row / column tails needs no predicates and three FP instructions per element.
    float* o = p.dst + (size_t)ma * p.out_ld + p.out_coff + n0 + 2 * q4;
    const float* rp = p.res ? p.res + (size_t)ma * p.res_ld + p.res_coff + n0 + 2 * q4 : nullptr;
    const size_t o8 = (size_t)8 * p.out_ld, r8 = (size_t)8 * p.res_ld;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * q4;
      float2 b2 = make_float2(0.f, 0.f), s2 = make_float2(1.f, 1.f), h2 = b2;
      if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + n));
      if (p.post_s) {
        s2 = __ldg(reinterpret_cast<const float2*>(p.post_s + n));
        h2 = __ldg(reinterpret_cast<const float2*>(p.post_h + n));
      }
      float2 rr[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
      if (rp) {
        rr[0] = __ldg(reinterpret_cast<const float2*>(rp + 8 * j));
        rr[1] = __ldg(reinterpret_cast<const float2*>(rp + 8 * j + r8));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 x = make_float2(res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
        x.x = fmaf(x.x, descale, b2.x); x.y = fmaf(x.y, descale, b2.y);      // descale == 1 on the tf32 path
        if (e.relu) { x.x = fminf(fmaxf(x.x, 0.f), e.hi1); x.y = fminf(fmaxf(x.y, 0.f), e.hi1); }
        if (p.post_s) { x.x = fmaf(x.x, s2.x, h2.x); x.y = fmaf(x.y, s2.y, h2.y); }
        if (rp) { x.x += rr[h].x; x.y += rr[h].y; }
        if (e.relu2) { x.x = fminf(fmaxf(x.x, 0.f), e.hi2); x.y = fminf(fmaxf(x.y, 0.f), e.hi2); }
        *reinterpret_cast<float2*>(o + 8 * j + h * o8) = x;
        tmax = fmaxf(tmax, fmaxf(fabsf(x.x), fabsf(x.y)));
      }
    }
    return;
  }
  // General epilogue: row / column tails and the per-utterance / gated / accumulate-into layers.
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + 2 * q4;
    if (n >= p.N) continue;              // N % 4 == 0: n < N implies n + 1 < N
    float2 b2 = make_float2(0.f, 0.f), s2 = make_float2(1.f, 1.f), h2 = b2;
    if (p.bias) b2 = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    if (p.post_s) {
      s2 = __ldg(reinterpret_cast<const float2*>(p.post_s + n));
      h2 = __ldg(reinterpret_cast<const float2*>(p.post_h + n));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = ma + 8 * h;
      if (m >= p.M) continue;
      float2 x = make_float2(res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
      // acc * descale + bias in one rounding (descale == 1 on the tf32 path: exactly acc + bias) -- the same
      // expression as the fast path, so a row's result does not depend on which path its tile took
      x.x = fmaf(x.x, descale, b2.x); x.y = fmaf(x.y, descale, b2.y);
      const int ur = e.need_urow ? urow_of(p, m) : 0;
      if (p.ubias) {
        const float2 u = __ldg(reinterpret_cast<const float2*>(p.ubias + (size_t)ur * p.N + n));
        x.x += u.x; x.y += u.y;
      }
      if (p.act == VP_ACT_RELU) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); }
      else if (p.act != VP_ACT_NONE) x = act2_slow(x, p.act);
      if (p.post_s) { x.x = fmaf(x.x, s2.x, h2.x); x.y = fmaf(x.y, s2.y, h2.y); }
      if (p.gate) {
        const float2 gt = __ldg(reinterpret_cast<const float2*>(p.gate + (size_t)ur * p.N + n));
        x.x *= gt.x; x.y *= gt.y;
      }
      if (p.res) {
        const float2 r = __ldg(reinterpret_cast<const float2*>(p.res + (size_t)m * p.res_ld + p.res_coff + n));
        x.x += r.x; x.y += r.y;
      }
      if (p.act2 == VP_ACT_RELU) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); }
      else if (p.act2 != VP_ACT_NONE) x = act2_slow(x, p.act2);
      *reinterpret_cast<float2*>(p.dst + (size_t)m * p.out_ld + p.out_coff + n) = x;
      tmax = fmaxf(tmax, fmaxf(fabsf(x.x), fabsf(x.y)));
      if (p.sum) {                         // accumulate-into view (Res2 chains): sum[m, n] += y[m, n]
        float2* sq = reinterpret_cast<float2*>(p.sum + (size_t)m * p.sum_ld + p.sum_coff + n);
        float2 sv = *sq;
        sv.x += x.x; sv.y += x.y;
        *sq = sv;
      }
    }
  }
}

template <int MODE> struct Slot;
template <> struct Slot<0> { float4 v[ROWS_PER_THREAD]; };
template <> struct Slot<1> { float4 v[ROWS_PER_THREAD]; float4 u[ROWS_PER_THREAD]; };
template <> struct Slot<2> { float4 v[ROWS_PER_THREAD]; float4 ps, ph; uint32_t okmask; };
struct SlotH { float4 v[ROWS_PER_THREAD]; float4 w[ROWS_PER_THREAD]; };   // F16 path: 8 consecutive K elements per row

struct TcArgs {
  const float* w_tc;     // pre-split, pre-tiled, pre-swizzled weights: [n_tile][k_block][hi BN x 128 B | lo BN x 128 B]
  int BN;                // N tile (multiple of 16, <= 128; <= 64 when n_chunks > 1)
  int stages;
  int m_tiles, n_tiles, k_blocks;
  int kc, n_chunks;      // K blocks per accumulation chunk / chunks per tile (long-K layers: bounded accumulation length)
  int debug;             // experiments only (VPB_TC_DEBUG): 1 = skip B copies, 2 = skip A global loads, 4 = skip MMAs
  float descale;         // F16 path only: 1 / (power-of-two scale folded into the fp16 weight image); keep LAST
};

// F16 = true (MODE 0 only): operands are split into two fp16 terms instead of two tf32 terms -- hi = fp16(x),
// lo = fp16(x - hi), same three MMAs, wgmma f16 at twice the tf32 rate; a stage row of 128 B then holds 64 K elements
// (BKE) and a producer thread moves 8 of them per row (KPT).
template <int MODE, bool F16, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvParams p,
                                                                 const __grid_constant__ TcArgs a) {
  static_assert(!F16 || MODE == 0, "the fp16 split path only implements the plain / concat source mode");
  static_assert(BN % 16 == 0 && BN >= 16 && BN <= MAX_BN, "N tile");
  constexpr bool CHUNKABLE = BN <= MAX_BN_CHUNKED;
  constexpr int BKE = F16 ? 64 : BK;     // K elements per pipeline stage
  constexpr int KPT = F16 ? 8 : 4;       // K elements per producer thread and row
  using SlotT = typename std::conditional<F16, SlotH, Slot<MODE>>::type;
  pdl_launch_dependents();                 // the next kernel's CTAs may be scheduled as SMs free up (see common.cuh)
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * 8];     // full[S], empty[S]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t b_tile = (uint32_t)BN * 128u;             // bytes of one (hi|lo) B tile
  constexpr uint32_t stage_bytes = 2u * A_TILE + 2u * b_tile;
  const int S = a.stages;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[8]);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, PRODUCER_WARPS + 1);            // one arrival per A-producer warp + 1 expect_tx arrival (B)
      mbar_init(empty0 + 8 * s, CONSUMER_WARPS);               // one arrival per consumer warp once its wgmmas retired
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // barrier init above overlaps the tail of the previous kernel; everything below touches activations / amax slots /
  // the output
  pdl_wait();

  // work distribution: tile g = (m_tile, n_tile), n fastest, strided over the persistent grid
  const int total_groups = a.m_tiles * a.n_tiles;

  if (warp >= CONSUMER_WARPS) {
    // =========================== A producers ===========================
    // Thread t owns the 16-byte chunk `chunk` of rows r0 + 32*i: a warp-level load covers 4 rows x 128 contiguous bytes.
    // All tap / channel arithmetic is per K block (uniform over the thread's rows); per row only the bounds test remains.
    const int t = threadIdx.x - CONSUMER_THREADS;
    const int chunk = t & 7;
    const int r0 = t >> 3;                 // 0..31
    const bool pointwise = (p.KT * p.KF == 1);
    // The (tile, K block) pairs of this CTA form ONE flat stream: the gather cursor runs DEPTH items ahead of the publish
    // cursor and crosses tile boundaries, so the load pipeline never drains between tiles.
    const int my_tiles = (total_groups - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_items = my_tiles * a.k_blocks;
    RowInfo rows[ROWS_PER_THREAD];
    // Gather cursor.  gather() is always called for consecutive items q = 0, 1, 2, ..., so the (tile, K block, tap,
    // channel) decomposition of q is kept incrementally -- no integer division per K block (the per-call divisions +
    // 64-bit row arithmetic made the producers instruction-issue bound at N = 64).
    int g_tl = 0, g_kb = 0;                    // tile (local index) and K block of the next item to gather
    int g_k = chunk * KPT;                     // this thread's first k of that K block
    int g_ci = 0, g_kt = 0, g_kf = 0;          // channel / tap position of g_k
    auto cursor_reset = [&]() {
      g_kb = 0; g_k = chunk * KPT; g_ci = g_k; g_kt = 0; g_kf = 0;
      if (!pointwise)
        while (g_ci >= p.CinTot) { g_ci -= p.CinTot; if (++g_kf == p.KF) { g_kf = 0; ++g_kt; } }
    };
    cursor_reset();
    {
      // Register prefetch slots.  gather() ONLY issues loads (no instruction may read a loaded register before publish():
      // even a predicated-off consumer stalls on the load's scoreboard and would serialise the loads); add / BN-ReLU
      // prologue are applied in publish().  MODE 0: plain or channel-concat source, 3 K blocks in flight; MODE 1: second
      // source added (x_i + y_{i-1}); MODE 2: per-channel affine(+ReLU) prologue; 2 K blocks in flight for 1 and 2.
      SlotT sl0, sl1, sl2;
      auto gather = [&](SlotT& sl) {
        if (g_kb == 0) {                       // cursor entered a new tile: decode its 4 rows
          const int g = (int)blockIdx.x + g_tl * (int)gridDim.x;
          const int m0 = (g / a.n_tiles) * BM;
#pragma unroll
          for (int i = 0; i < ROWS_PER_THREAD; ++i) {
            rows[i] = decode_row(p, m0 + r0 + 32 * i);
            if (!rows[i].valid) rows[i].t0 = -(1 << 28);        // fails every bounds test below (also after reflection)
          }
        }
        const int ci = g_ci;
        const int dt = g_kt * p.dT, df = g_kf * p.dF;
        const bool kok = g_k < p.K && !(a.debug & 2);
        const bool second = (MODE == 0) && (p.src2_mode == VP_SRC2_CONCAT) && (ci >= p.Cin);
        const char* base = reinterpret_cast<const char*>(second ? p.src2 + p.src2_coff + (ci - p.Cin) : p.src + p.in_coff + ci);
        const uint32_t ldb = (uint32_t)(second ? p.src2_ld : p.in_ld) * 4u;      // row pitch in bytes
        if constexpr (MODE == 2) {
          sl.ps = make_float4(1.f, 1.f, 1.f, 1.f);
          sl.ph = make_float4(0.f, 0.f, 0.f, 0.f);
          if (kok) {
            sl.ps = __ldg(reinterpret_cast<const float4*>(p.pre_s + ci));
            sl.ph = __ldg(reinterpret_cast<const float4*>(p.pre_h + ci));
          }
          sl.okmask = 0;
        }
#pragma unroll
        for (int i = 0; i < ROWS_PER_THREAD; ++i) {
          int ti = rows[i].t0 + dt;
          const int fi = rows[i].f0 + df;
          if (p.pad_mode == VP_PAD_REFLECT) {
            if (ti < 0) ti = -ti;
            if (ti >= p.Tin) ti = 2 * (p.Tin - 1) - ti;
          }
          const bool ok = kok && (unsigned)ti < (unsigned)p.Tin && (unsigned)fi < (unsigned)p.Fin;
          const uint32_t r = (uint32_t)(rows[i].base + ti * p.Fin + fi);       // source row index (< 2^31 rows)
          sl.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok) sl.v[i] = __ldg(reinterpret_cast<const float4*>(base + (uint64_t)r * ldb));
          if constexpr (F16) {
            sl.w[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) sl.w[i] = __ldg(reinterpret_cast<const float4*>(base + (uint64_t)r * ldb + 16));
          }
          if constexpr (MODE == 1) {
            sl.u[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok)
              sl.u[i] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const char*>(p.src2 + p.src2_coff + ci) +
                                                              (uint64_t)r * ((uint32_t)p.src2_ld * 4u)));
          }
          if constexpr (MODE == 2) sl.okmask |= ok ? (1u << i) : 0u;
        }
        // advance the cursor by one K block
        if (++g_kb == a.k_blocks) {
          ++g_tl;
          cursor_reset();
        } else {
          g_k += BKE;
          g_ci += BKE;
          if (!pointwise)
            while (g_ci >= p.CinTot) { g_ci -= p.CinTot; if (++g_kf == p.KF) { g_kf = 0; ++g_kt; } }
        }
      };
      constexpr int DEPTH = (MODE == 0 && !F16) ? 3 : 2;
      int p_s = 0;
      uint32_t p_ph = 0;
      // fp16 split: dynamic power-of-two activation scale from the source tensor's amax slot (written by the ops that
      // produced the tensor, complete at kernel start) -> |x * ascale| < 2^14, range-safe for any activation magnitude
      float ascale = 1.f;
      if constexpr (F16) ascale = exp2i(f16_scale_exp(__ldg(p.amax_in)));
      auto publish = [&](int q, SlotT& sl) {
        const int s = p_s;
        const uint32_t ph = p_ph;
        if (++p_s == S) { p_s = 0; p_ph ^= 1u; }
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        if (t == 0) {                        // B: one bulk copy of the stage's weight image (item q = tile, K block)
          if (a.debug & 1) {
            mbar_arrive(full0 + 8 * s);
          } else {
            const int tl = q / a.k_blocks, kb = q - tl * a.k_blocks;
            const int nt = ((int)blockIdx.x + tl * (int)gridDim.x) % a.n_tiles;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(a.w_tc) + ((size_t)nt * a.k_blocks + kb) * (2u * b_tile);
            mbar_expect_tx(full0 + 8 * s, 2u * b_tile);
            bulk_copy_g2s(smem_base + s * stage_bytes + 2u * A_TILE, src, 2u * b_tile, full0 + 8 * s);
          }
        }
        const uint32_t a_hi = smem_base + s * stage_bytes;
        const uint32_t a_lo = a_hi + A_TILE;
#pragma unroll
        for (int i = 0; i < ROWS_PER_THREAD; ++i) {
          const int r = r0 + 32 * i;
          const uint32_t off = (uint32_t)r * 128u + (uint32_t)((chunk ^ (r & 7)) << 4);
          if constexpr (F16) {
            // 8 consecutive K elements -> one 16-byte chunk of fp16 hi and one of fp16 lo (lo = x - hi, exact in fp32)
            const float xs[8] = {sl.v[i].x * ascale, sl.v[i].y * ascale, sl.v[i].z * ascale, sl.v[i].w * ascale,
                                 sl.w[i].x * ascale, sl.w[i].y * ascale, sl.w[i].z * ascale, sl.w[i].w * ascale};
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const __half2 h = __floats2half2_rn(xs[2 * j], xs[2 * j + 1]);
              const float2 hf = __half22float2(h);
              const __half2 l = __floats2half2_rn(xs[2 * j] - hf.x, xs[2 * j + 1] - hf.y);
              hw[j] = *reinterpret_cast<const uint32_t*>(&h);
              lw[j] = *reinterpret_cast<const uint32_t*>(&l);
            }
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a_hi + off), "r"(hw[0]), "r"(hw[1]), "r"(hw[2]), "r"(hw[3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a_lo + off), "r"(lw[0]), "r"(lw[1]), "r"(lw[2]), "r"(lw[3]) : "memory");
            continue;
          }
          float4 x = sl.v[i];
          if constexpr (MODE == 1) { x.x += sl.u[i].x; x.y += sl.u[i].y; x.z += sl.u[i].z; x.w += sl.u[i].w; }
          if constexpr (MODE == 2) {
            if (sl.okmask & (1u << i)) {              // zero padding stays zero: the conv pads the BN-ReLU'd map
              x.x = fmaf(x.x, sl.ps.x, sl.ph.x); x.y = fmaf(x.y, sl.ps.y, sl.ph.y);
              x.z = fmaf(x.z, sl.ps.z, sl.ph.z); x.w = fmaf(x.w, sl.ps.w, sl.ph.w);
              if (p.pre_relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
            }
          }
          float4 hi, lo;
          hi.x = tf32_rna(x.x); hi.y = tf32_rna(x.y); hi.z = tf32_rna(x.z); hi.w = tf32_rna(x.w);
          lo.x = x.x - hi.x; lo.y = x.y - hi.y; lo.z = x.z - hi.z; lo.w = x.w - hi.w;
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a_hi + off), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a_lo + off), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
        }
        fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(full0 + 8 * s);     // one arrival per producer warp
        if (q + DEPTH < total_items) gather(sl);   // refill this slot (item q + DEPTH): DEPTH K blocks of loads stay in flight
      };
      if (total_items > 0) gather(sl0);
      if (total_items > 1) gather(sl1);
      if constexpr (DEPTH == 3) {
        if (total_items > 2) gather(sl2);
        for (int q = 0; q < total_items; q += 3) {
          publish(q, sl0);
          if (q + 1 < total_items) publish(q + 1, sl1);
          if (q + 2 < total_items) publish(q + 2, sl2);
        }
      } else {
        for (int q = 0; q < total_items; q += 2) {
          publish(q, sl0);
          if (q + 1 < total_items) publish(q + 1, sl1);
        }
      }
    }
  } else {
    // =========================== consumers: wgmma + epilogue ===========================
    const int wg = warp >> 2;                // warpgroup: tile rows 64*wg ..
    const int q4 = lane & 3;                 // fragment: columns 8j + 2*q4 (+1)
    const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // fragment rows rbase and rbase + 8 of the tile
    float acc[BN / 2];
    float run[BN / 2];                       // running sum of the finished accumulation chunks (CHUNKABLE only)
    float (&res)[BN / 2] = *(CHUNKABLE ? &run : &acc);     // what the epilogue reads
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0;
    uint32_t sph = 0;                                         // stage / phase cursors, advanced without divisions
    float descale = 1.f;                                      // fp16 split: 2^-k of the weight image x 2^-s of the activation scale
    if constexpr (F16) descale = a.descale * exp2i(-f16_scale_exp(__ldg(p.amax_in)));
    float tmax = 0.f;                                         // running max |y| of everything this thread stores (amax_out slot)
    const Epi epi = make_epi(p, descale);
    for (int g = blockIdx.x; g < total_groups; g += gridDim.x) {
      const int m0 = (g / a.n_tiles) * BM;
      const int n0 = (g % a.n_tiles) * BN;
      if (g + (int)gridDim.x < total_groups) prefetch_res<BN>(p, g + gridDim.x, a.n_tiles, warp, lane);
      // Long-K layers are accumulated in chunks of `kc` K blocks, each into a fresh accumulator that is then folded
      // into a running fp32 sum with correctly rounded adds.  (The tensor core truncates on every accumulate; the bias
      // grows linearly with the number of accumulates.)
      for (int ch = 0; ch < a.n_chunks; ++ch) {
        const int kb0 = ch * a.kc;
        const int kb1 = (kb0 + a.kc < a.k_blocks) ? kb0 + a.kc : a.k_blocks;
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(full0 + 8 * s, sph);
          const uint32_t a_hi = smem_base + s * stage_bytes + wg * (A_TILE / 2), a_lo = a_hi + A_TILE;
          const uint32_t b_hi = smem_base + s * stage_bytes + 2u * A_TILE, b_lo = b_hi + b_tile;
          wgmma_fence();
          if (!(a.debug & 4)) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {       // tf32: K = 8 / f16: K = 16 per instruction = 32 bytes of the row
              const uint32_t first = (kb != kb0) || (kk != 0);
              mma_tile<BN, F16>(acc, a_lo + kk * 32, b_hi + kk * 32, first);
              mma_tile<BN, F16>(acc, a_hi + kk * 32, b_lo + kk * 32, 1);
              mma_tile<BN, F16>(acc, a_hi + kk * 32, b_hi + kk * 32, 1);
            }
          }
          wgmma_commit();
          if (prev >= 0) {                     // the previous K block's group has retired: release its stage
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(empty0 + 8 * prev);
          }
          prev = s;
          if (++s == S) { s = 0; sph ^= 1u; }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
        if constexpr (CHUNKABLE) {
          {
            if (ch == 0) {
#pragma unroll
              for (int i = 0; i < BN / 2; ++i) run[i] = acc[i];
            } else {
#pragma unroll
              for (int i = 0; i < BN / 2; ++i) run[i] = acc[i] + run[i];
            }
          }
        }
      }
      store_tile<BN>(p, epi, res, m0, n0, m0 + rbase, q4, tmax);
    }
    if (p.amax_out) amax_commit(p.amax_out, tmax);     // one atomicMax per consumer warp per launch
  }
}

// per (kernel instantiation, device): opt into the dynamic shared memory, then launch
template <int MODE, bool F16, int BN>
static cudaError_t launch_bn(const cudaLaunchConfig_t& cfg, const ConvParams& p, const TcArgs& a) {
  static PerDeviceSmem once;
  if (once.need(cfg.dynamicSmemBytes)) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<MODE, F16, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)cfg.dynamicSmemBytes);
    if (e != cudaSuccess) return e;
    once.set(cfg.dynamicSmemBytes);
  }
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel<MODE, F16, BN>, p, a);
}

template <int MODE, bool F16>
static cudaError_t launch_mode(const cudaLaunchConfig_t& cfg, const ConvParams& p, const TcArgs& a) {
  if constexpr (F16) {                      // fp16 split: N >= 128 only (conv_tc16_supported) -> tiles of 128 or 64
    if (a.BN == 128) return launch_bn<MODE, F16, 128>(cfg, p, a);
    if (a.BN == 64) return launch_bn<MODE, F16, 64>(cfg, p, a);
    return cudaErrorInvalidConfiguration;
  } else {
    switch (a.BN) {
      case 16: return launch_bn<MODE, F16, 16>(cfg, p, a);
      case 32: return launch_bn<MODE, F16, 32>(cfg, p, a);
      case 48: return launch_bn<MODE, F16, 48>(cfg, p, a);
      case 64: return launch_bn<MODE, F16, 64>(cfg, p, a);
      case 80: return launch_bn<MODE, F16, 80>(cfg, p, a);
      case 96: return launch_bn<MODE, F16, 96>(cfg, p, a);
      case 112: return launch_bn<MODE, F16, 112>(cfg, p, a);
      case 128: return launch_bn<MODE, F16, 128>(cfg, p, a);
      default: return cudaErrorInvalidConfiguration;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Wide FP16-split path for pointwise convs (launch_conv_tc16, tc16_wide_ok): 128 x 256 output tiles.
//
// The 128 x 128 kernel above pulls 64 KB from the L2 per 2.1 MFLOP stage (A as fp32 gathered by 256 producer threads,
// B as the hi|lo fp16 image) and is L2-bandwidth bound.  A pointwise conv's A tile is a plain 2-D box of the channel-last
// [M, K] view, so here one thread loads it with TMA (zero fill gives the M and K tails), the consumer warps split it into
// fp16 hi / lo in registers (the same arithmetic as publish() above) and issue wgmma with A from registers, and the freed
// registers hold a 256-wide accumulator: 96 KB of L2 traffic per 4.2 MFLOP stage.
//   warps 0-7  consumers : two warpgroups of 64 rows, 232 registers each (setmaxnreg), 128 fp32 accumulators
//   warps 8-11 producer  : one thread issues the stage's two A boxes and four B copies onto the stage's `full` mbarrier
// B stage = n-tiles 2j and 2j + 1 of the 128-wide fp16 image at the same K block: hi | hi | lo | lo, so that B_hi and B_lo
// each are 256 contiguous swizzled rows.  The three MMAs per K16 step run in the order of the 128-wide kernel
// (A_lo B_hi, A_hi B_lo, A_hi B_hi) into one accumulator, so its first 128 columns equal that kernel's bit for bit.
constexpr int WBN = 256;
constexpr int W_A_BOX = BM * 128;                 // 16 KB: one TMA box of 128 rows x 32 fp32 (one SWIZZLE_128B row each)
constexpr int W_A_STAGE = 2 * W_A_BOX;            // 64 K elements of fp32 A
constexpr int W_B_HALF = WBN * 128;               // 32 KB: 256 rows x 64 fp16 (B_hi or B_lo)
constexpr int W_STAGE = W_A_STAGE + 2 * W_B_HALF; // 96 KB
constexpr int W_STAGES = 2;
constexpr int W_THREADS = CONSUMER_THREADS + 128;
constexpr int W_SMEM = W_STAGES * W_STAGE + 1024;

struct WideArgs {
  const uint8_t* w_tc16;  // the 128-wide fp16 image: [n_tile][k_block][hi 128 x 128 B | lo 128 x 128 B]
  int m_tiles, n_tiles, k_blocks;  // n_tiles of 256 columns; k_blocks of 64
  float descale;
};

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}

// fp32 pair -> fp16 hi and lo terms of x * ascale, op for op as publish() above
__device__ __forceinline__ void split_f16(float2 x, float ascale, uint32_t& hw, uint32_t& lw) {
  const float x0 = x.x * ascale, x1 = x.y * ascale;
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hw = *reinterpret_cast<const uint32_t*>(&h);
  lw = *reinterpret_cast<const uint32_t*>(&l);
}

// One consumer warpgroup's K block (64 K = 4 x K16) of a stage: load its 64 rows of fp32 A from the swizzled stage,
// split, and issue the 12 wgmmas as one group.  ah / al must stay untouched until that group has retired.
__device__ __forceinline__ void wide_kblock(float (&acc)[WBN / 2], uint32_t (&ah)[4][4], uint32_t (&al)[4][4],
                                            uint32_t a_rows, uint32_t b_hi, int q4, float ascale, bool first) {
  const uint32_t sw = a_rows >> 7 & 7;   // the fragment's rows r and r + 8 share r & 7
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t half = a_rows + (kk >> 1) * W_A_BOX;
    const uint32_t c = (kk & 1) * 4 + (q4 >> 1);         // 16-byte chunk of columns 16 (kk & 1) + 2 q4 (+1)
    const uint32_t lo8 = (q4 & 1) * 8;
    float2 x[4];
    // (r, c), (r + 8, c), (r, c + 8 columns = 2 chunks), (r + 8, c + 2 chunks)
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x[0].x), "=f"(x[0].y) : "r"(half + ((c ^ sw) << 4) + lo8));
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x[1].x), "=f"(x[1].y) : "r"(half + 1024 + ((c ^ sw) << 4) + lo8));
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x[2].x), "=f"(x[2].y) : "r"(half + (((c + 2) ^ sw) << 4) + lo8));
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x[3].x), "=f"(x[3].y) : "r"(half + 1024 + (((c + 2) ^ sw) << 4) + lo8));
#pragma unroll
    for (int i = 0; i < 4; ++i) split_f16(x[i], ascale, ah[kk][i], al[kk][i]);
  }
  wgmma_fence();
  const uint32_t b_lo = b_hi + W_B_HALF;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    wgmma_f16_rs_n256(acc, al[kk], smem_desc(b_hi + kk * 32), (first && kk == 0) ? 0u : 1u);
    wgmma_f16_rs_n256(acc, ah[kk], smem_desc(b_lo + kk * 32), 1u);
    wgmma_f16_rs_n256(acc, ah[kk], smem_desc(b_hi + kk * 32), 1u);
  }
  wgmma_commit();
}

__global__ void __launch_bounds__(W_THREADS, 1) conv_tc16_wide_kernel(const __grid_constant__ ConvParams p,
                                                                      const __grid_constant__ WideArgs a,
                                                                      const __grid_constant__ CUtensorMap amap) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bars[2 * W_STAGES];     // full[S], empty[S]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[W_STAGES]);
  if (threadIdx.x == 0) {
    for (int s = 0; s < W_STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);                        // the producer's expect_tx arrival; TMA completes the bytes
      mbar_init(empty0 + 8 * s, CONSUMER_WARPS);          // one arrival per consumer warp once its wgmmas retired
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  const int total = a.m_tiles * a.n_tiles;

  if (warp >= CONSUMER_WARPS) {
    // =========================== producer ===========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
    if (warp != CONSUMER_WARPS || lane != 0) return;
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&amap)) : "memory");
    constexpr uint32_t img_half = 128u * 128u;                 // hi (or lo) of one 128-wide image tile
    int s = 0;
    uint32_t ph = 0;
    for (int g = blockIdx.x; g < total; g += gridDim.x) {
      const int m0 = (g / a.n_tiles) * BM;
      const int nt = g % a.n_tiles;
      for (int kb = 0; kb < a.k_blocks; ++kb) {
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        const uint32_t st = smem_base + s * W_STAGE, bar = full0 + 8 * s;
        mbar_expect_tx(bar, W_STAGE);
        tma_load_2d(st, &amap, kb * 64, m0, bar);
        tma_load_2d(st + W_A_BOX, &amap, kb * 64 + 32, m0, bar);
        const uint8_t* t0 = a.w_tc16 + ((size_t)(2 * nt) * a.k_blocks + kb) * (2u * img_half);
        const uint8_t* t1 = t0 + (size_t)a.k_blocks * (2u * img_half);   // n-tile 2 nt + 1, same K block
        const uint32_t b = st + W_A_STAGE;
        bulk_copy_g2s(b, t0, img_half, bar);
        bulk_copy_g2s(b + img_half, t1, img_half, bar);
        bulk_copy_g2s(b + W_B_HALF, t0 + img_half, img_half, bar);
        bulk_copy_g2s(b + W_B_HALF + img_half, t1 + img_half, img_half, bar);
        if (++s == W_STAGES) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }
  // =========================== consumers: split + wgmma + epilogue ===========================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
  const int wg = warp >> 2;
  const int q4 = lane & 3;
  const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // fragment rows rbase and rbase + 8 of the tile
  const int sexp = f16_scale_exp(__ldg(p.amax_in));
  const float ascale = exp2i(sexp);
  const Epi epi = make_epi(p, a.descale * exp2i(-sexp));
  float acc[WBN / 2];
#pragma unroll
  for (int i = 0; i < WBN / 2; ++i) acc[i] = 0.f;
  // two fragment sets, alternating by K block: a K block's set is rewritten only after wgmma_wait<1> in the next K block
  // has retired the group that read it
  uint32_t ah0[4][4], al0[4][4], ah1[4][4], al1[4][4];
  float tmax = 0.f;
  int s = 0;
  uint32_t sph = 0;
  for (int g = blockIdx.x; g < total; g += gridDim.x) {
    const int m0 = (g / a.n_tiles) * BM;
    const int n0 = (g % a.n_tiles) * WBN;
    if (g + (int)gridDim.x < total) prefetch_res<WBN>(p, g + gridDim.x, a.n_tiles, warp, lane);
    int prev = -1;
    for (int kb = 0; kb < a.k_blocks; ++kb) {
      mbar_wait(full0 + 8 * s, sph);
      const uint32_t st = smem_base + s * W_STAGE;
      const uint32_t a_rows = st + (uint32_t)rbase * 128u;
      if (kb & 1) wide_kblock(acc, ah1, al1, a_rows, st + W_A_STAGE, q4, ascale, false);
      else wide_kblock(acc, ah0, al0, a_rows, st + W_A_STAGE, q4, ascale, kb == 0);
      if (prev >= 0) {                     // the previous K block's group has retired: release its stage
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty0 + 8 * prev);
      }
      prev = s;
      if (++s == W_STAGES) { s = 0; sph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
    store_tile<WBN>(p, epi, acc, m0, n0, m0 + rbase, q4, tmax);
  }
  if (p.amax_out) amax_commit(p.amax_out, tmax);     // one atomicMax per consumer warp per launch
}

}  // namespace tc

// Host-visible tiling rule (mirrored by the Python packer mvector/engine.py::tc_tile_n).  The accumulator lives in the
// consumer threads' registers: 128-wide tiles, and 64-wide for chunked layers (vp_op.tc_kc > 0), which keep a second
// register set for the running sum.
static int tc_tile_n(int N, bool chunked) {
  const int cap = chunked ? tc::MAX_BN_CHUNKED : tc::MAX_BN;
  return N >= cap ? cap : (N + 15) & ~15;
}

bool conv_tc_supported(const ConvParams& p) {
  if (p.w_tc == nullptr) return false;
  if (p.M < 1024) return false;                       // tiny-M ops (SE / ASP bias / final FC) stay on the exact FFMA engine
  if (p.N < 16 || (p.N & 3) || (p.K & 3)) return false;
  if (p.tc_kc < 0 || (p.tc_kc & 63)) return false;
  if (p.tc_bn != tc_tile_n(p.N, p.tc_kc > 0)) return false;
  // the BN-ReLU prologue gather (MODE 2) reads one source only: prologue + second source stays on the FFMA engine, whose
  // gather composes both (common.cuh::gather_a4)
  if (p.pre_s != nullptr && p.src2_mode != VP_SRC2_NONE) return false;
  return true;
}

// persistent grids: one CTA per SM of the current device
static int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  static int count[64] = {};
  if (dev >= 0 && dev < 64) {
    if (count[dev] == 0) cudaDeviceGetAttribute(&count[dev], cudaDevAttrMultiProcessorCount, dev);
    if (count[dev] > 0) sms = count[dev];
  }
  return sms;
}

// f16 = true: two-term FP16 split (conv_tc_kernel<0, true, BN>); w_img is then the fp16 weight image and descale the
// inverse of the power-of-two scale folded into it.
static cudaError_t launch_conv_tc_impl(const ConvParams& p, const float* w_img, bool f16, float descale, cudaStream_t stream) {
  using namespace tc;
  TcArgs a;
  a.w_tc = w_img;
  a.descale = descale;
  a.BN = p.tc_bn;
  const int bke = f16 ? 64 : BK;
  const int stage_bytes = 2 * A_TILE + 2 * a.BN * 128;
  a.stages = SMEM_BUDGET / stage_bytes;
  if (a.stages > 8) a.stages = 8;
  if (a.stages < 2) return cudaErrorInvalidConfiguration;
  a.m_tiles = (p.M + BM - 1) / BM;
  a.n_tiles = (p.N + a.BN - 1) / a.BN;
  a.k_blocks = (p.K + bke - 1) / bke;
  a.kc = (p.tc_kc > 0 && p.tc_kc < p.K) ? p.tc_kc / bke : a.k_blocks;
  a.n_chunks = (a.k_blocks + a.kc - 1) / a.kc;
  if (a.n_chunks > 1 && a.BN > MAX_BN_CHUNKED) return cudaErrorInvalidConfiguration;
  static int debug_flags = -1;
  if (debug_flags < 0) { const char* e = getenv("VPB_TC_DEBUG"); debug_flags = e ? atoi(e) : 0; }
  a.debug = debug_flags;
  const int sms = sm_count();
  const int groups = a.m_tiles * a.n_tiles;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sms < groups ? sms : groups);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = (size_t)a.stages * stage_bytes + 1024;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e;
  if (f16) e = launch_mode<0, true>(cfg, p, a);
  else if (p.pre_s != nullptr) e = launch_mode<2, false>(cfg, p, a);
  else if (p.src2_mode == VP_SRC2_ADD) e = launch_mode<1, false>(cfg, p, a);
  else e = launch_mode<0, false>(cfg, p, a);
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
}

cudaError_t launch_conv_tc(const ConvParams& p, cudaStream_t stream) {
  return launch_conv_tc_impl(p, p.w_tc, false, 1.f, stream);
}

// FP16-split engine: plain / concat source only, 8-element channel granularity, the same tiling rule as the tf32 image,
// and a source tensor whose amax slot is tracked (dynamic power-of-two activation scale -> range-safe).
bool conv_tc16_supported(const ConvParams& p) {
  if (!conv_tc_supported(p)) return false;
  if (p.amax_in == nullptr) return false;
  if (p.pre_s != nullptr || p.src2_mode == VP_SRC2_ADD) return false;
  if ((p.Cin & 7) || (p.CinTot & 7) || (p.K & 7)) return false;
  return p.N >= 128;                                  // narrow layers are not tensor bound: nothing to gain
}

// The wide path (conv_tc16_wide_kernel): a pointwise, stride-1, unpadded conv reading one plain source, unchunked, whose
// A view [M, K] (base src + in_coff, row pitch in_ld) is a legal TMA tensor and whose N splits into 256-wide tiles.
// N >= 1024 only: at N = 512 (ECAPA's tdnn1 / tdnn2, M = 76 288) the wide kernel measured 4 % slower than the 128-wide
// one (9.03 waves of 256-wide tiles on 132 SMs against 19 of 128-wide ones), at N = 1536 it is faster.
static bool tc16_wide_ok(const ConvParams& p) {
  if (p.KT != 1 || p.KF != 1 || p.sT != 1 || p.sF != 1 || p.padT != 0 || p.padF != 0) return false;
  if (p.Tin != p.Tout || p.Fin != p.Fout) return false;       // output row m reads source row m
  if (p.src2_mode != VP_SRC2_NONE || p.tc_kc != 0) return false;
  if (p.N % tc::WBN != 0 || p.N < 1024) return false;
  if ((p.in_ld & 3) || (p.in_coff & 3) || (p.out_ld & 3) || (p.out_coff & 3)) return false;
  return ((uintptr_t)(p.src + p.in_coff) & 15) == 0;
}

static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn == nullptr) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  }
  return fn;
}

static cudaError_t launch_conv_tc16_wide(const ConvParams& p, const float* w_tc16, float descale, cudaStream_t stream) {
  using namespace tc;
  PFN_cuTensorMapEncodeTiled_v12000 encode = tensor_map_encoder();
  if (encode == nullptr) return cudaErrorNotSupported;
  // A = the [M, K] fp32 view, boxes of 32 columns (128 B, one SWIZZLE_128B row) x 128 rows; reads outside it are zeros
  CUtensorMap amap;
  const cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.M};
  const cuuint64_t strides[1] = {(cuuint64_t)p.in_ld * 4u};
  const cuuint32_t box[2] = {32u, (cuuint32_t)BM};
  const cuuint32_t elem[2] = {1u, 1u};
  if (encode(&amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(p.src + p.in_coff), dims, strides, box, elem,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorInvalidValue;
  WideArgs a;
  a.w_tc16 = reinterpret_cast<const uint8_t*>(w_tc16);
  a.m_tiles = (p.M + BM - 1) / BM;
  a.n_tiles = p.N / WBN;
  a.k_blocks = (p.K + 63) / 64;
  a.descale = descale;
  const int groups = a.m_tiles * a.n_tiles;
  const int sms = sm_count();
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sms < groups ? sms : groups);
  cfg.blockDim = dim3(W_THREADS);
  cfg.dynamicSmemBytes = W_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  static PerDeviceSmem once;
  if (once.need(cfg.dynamicSmemBytes)) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc16_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM);
    if (e != cudaSuccess) return e;
    once.set(cfg.dynamicSmemBytes);
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, conv_tc16_wide_kernel, p, a, amap);
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
}

cudaError_t launch_conv_tc16(const ConvParams& p, const float* w_tc16, float descale, cudaStream_t stream) {
  if (tc16_wide_ok(p)) return launch_conv_tc16_wide(p, w_tc16, descale, stream);
  return launch_conv_tc_impl(p, w_tc16, true, descale, stream);
}

}  // namespace vpb
