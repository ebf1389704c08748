// Shared device helpers and kernel parameter blocks for the vpb200 library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "../../include/vpb200.h"

namespace vpb {

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) applies to the CURRENT device only: launchers remember, per device,
// the largest dynamic shared-memory size they have opted a kernel into.
struct PerDeviceSmem {
  size_t cfg[64] = {};
  // true when the kernel must be (re)configured on the current device before launching with `bytes` of dynamic smem
  bool need(size_t bytes, int* dev_out = nullptr) {
    int d = 0;
    cudaGetDevice(&d);
    if (dev_out) *dev_out = d;
    if (d < 0 || d >= 64) return bytes > 48 * 1024;
    return bytes > 48 * 1024 && bytes > cfg[d];
  }
  void set(size_t bytes) {
    int d = 0;
    cudaGetDevice(&d);
    if (d >= 0 && d < 64 && bytes > cfg[d]) cfg[d] = bytes;
  }
};

// ---- programmatic dependent launch (PDL) ----
// Every kernel of the library starts with pdl_launch_dependents() -- the next kernel in the stream may be scheduled as
// soon as all CTAs of this grid have started -- and calls pdl_wait() before its first access to mutable global memory
// (activations, features, amax slots; weights / constant tables are immutable).  pdl_wait() returns when the
// predecessor grid has COMPLETED and flushed, and the predecessor itself only completed after its own wait, so the
// ordering of a stream of such kernels is transitive: all that overlaps is a kernel's prologue (block scheduling,
// barrier set-up, parameter loads) with the tail of the kernel before it.  Without the launch attribute both
// instructions are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// VPB_PDL=0 launches everything fully serialised (per-kernel timing)
inline int pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("VPB_PDL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on;
}

// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-stream-serialisation attribute
template <typename K, typename... A>
inline void launch_pdl(K kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kern, args...);      // errors are picked up by the caller's cudaGetLastError()
}

// Resolved (device-pointer) form of a vp_op, passed to kernels by value.
struct ConvParams {
  const float* src; const float* src2; float* dst; float* sum; const float* res; const float* gate; const float* ubias;
  const float* w; const float* w_tc; const float* bias; const float* pre_s; const float* pre_h; const float* post_s; const float* post_h;
  int M, N, K;                       // M = B*Tout*Fout rows, N = Cout, K = KT*KF*CinTot
  int B, Tin, Fin, Cin, CinTot, in_ld, in_coff;
  int src2_mode, src2_ld, src2_coff;
  int Tout, Fout, out_ld, out_coff, res_ld, res_coff;
  int KT, KF, sT, sF, dT, dF, padT, padF, pad_mode;
  int w_ld, pre_relu, act, act2, seg_len, n_seg, tc_bn, tc_kc, sum_ld, sum_coff;
  unsigned* amax_out;                // slot this op maxes |y| into (or null)
  const unsigned* amax_in;           // slot holding max |x| of the source tensor (fp16 split only, else null)
};

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case VP_ACT_RELU: return fmaxf(v, 0.f);
    case VP_ACT_HARDTANH20: return fminf(fmaxf(v, 0.f), 20.f);
    case VP_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case VP_ACT_TANH: return tanhf(v);
    case VP_ACT_SILU: return v / (1.f + expf(-v));
    default: return v;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- amax slots (dynamic activation range of the fp16 split; include/vpb200.h vp_op.amax_out / amax_in) ----
// |v| as float bits order like unsigned integers, so one atomicMax per warp keeps the running maximum; max is exact and
// order independent, hence deterministic.
__device__ __forceinline__ float amax4(float m, const float4& v) {
  return fmaxf(fmaxf(m, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
}
__device__ __forceinline__ void amax_commit(unsigned* slot, float m) {     // whole warp must call
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(slot, __float_as_uint(m));
}
// Same for kernels with thousands of CTAs: reduce over the whole block first -- one atomic per CTA, not per warp (38 k
// atomics on one address cost the ew kernel 13 us in round 2).  Every thread of the block must call; blockDim <= 1024.
__device__ __forceinline__ void amax_commit_block(unsigned* slot, float m) {
  __shared__ float amax_red[32];
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) amax_red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int nw = (blockDim.x + 31) >> 5;
    float v = threadIdx.x < nw ? amax_red[threadIdx.x] : 0.f;
    v = warp_max(v);
    if (threadIdx.x == 0 && v > 0.f) atomicMax(slot, __float_as_uint(v));
  }
}

// exponent s such that amax * 2^s lies in [2^13, 2^14): fp16 hi terms stay below 65504, lo terms above the subnormals
__device__ __forceinline__ int f16_scale_exp(unsigned amax_bits) {
  const int be = (int)((amax_bits >> 23) & 0xffu);
  if (amax_bits == 0u || be == 0xff) return 0;          // all-zero tensor, or inf / nan (propagates like the reference)
  int s = 13 - (be - 127);
  return s < -100 ? -100 : (s > 100 ? 100 : s);
}
__device__ __forceinline__ float exp2i(int s) { return __uint_as_float((unsigned)(s + 127) << 23); }

// Decoded A-operand row (one output position): where its receptive field starts in the source map.
struct RowInfo {
  int base;   // b * Tin * Fin (row index of the utterance's first source row)
  int t0;     // to*sT - padT
  int f0;     // fo*sF - padF
  int valid;  // m < M
};

__device__ __forceinline__ RowInfo decode_row(const ConvParams& p, int m) {
  RowInfo r;
  r.valid = m < p.M;
  int mm = r.valid ? m : 0;
  int per = p.Tout * p.Fout;
  int b = mm / per;
  int rem = mm - b * per;
  int to = rem / p.Fout;
  int fo = rem - to * p.Fout;
  r.base = b * p.Tin * p.Fin;
  r.t0 = to * p.sT - p.padT;
  r.f0 = fo * p.sF - p.padF;
  return r;
}

// Gather 4 consecutive K elements (one tap, 4 channels) of the implicit-GEMM A operand, with zero / reflect padding,
// optional second source (add / channel-concat) and optional per-channel affine(+ReLU) prologue.
// k must be a multiple of 4; Cin, CinTot, in_ld, in_coff (and the src2 equivalents) multiples of 4.
__device__ __forceinline__ float4 gather_a4(const ConvParams& p, const RowInfo& r, int k) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!r.valid || k >= p.K) return v;
  int tap = k / p.CinTot;
  int ci = k - tap * p.CinTot;
  int kt = tap / p.KF;
  int kf = tap - kt * p.KF;
  int ti = r.t0 + kt * p.dT;
  int fi = r.f0 + kf * p.dF;
  if (p.pad_mode == VP_PAD_REFLECT) {
    if (ti < 0) ti = -ti;
    if (ti >= p.Tin) ti = 2 * (p.Tin - 1) - ti;
  }
  if (ti < 0 || ti >= p.Tin || fi < 0 || fi >= p.Fin) return v;
  size_t row = (size_t)r.base + (size_t)ti * p.Fin + fi;
  if (p.src2_mode == VP_SRC2_CONCAT && ci >= p.Cin) {
    v = __ldg(reinterpret_cast<const float4*>(p.src2 + row * p.src2_ld + p.src2_coff + (ci - p.Cin)));
  } else {
    v = __ldg(reinterpret_cast<const float4*>(p.src + row * p.in_ld + p.in_coff + ci));
    if (p.src2_mode == VP_SRC2_ADD) {
      float4 u = __ldg(reinterpret_cast<const float4*>(p.src2 + row * p.src2_ld + p.src2_coff + ci));
      v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
    }
  }
  if (p.pre_s != nullptr) {
    float4 s = __ldg(reinterpret_cast<const float4*>(p.pre_s + ci));
    float4 h = __ldg(reinterpret_cast<const float4*>(p.pre_h + ci));
    v.x = fmaf(v.x, s.x, h.x); v.y = fmaf(v.y, s.y, h.y); v.z = fmaf(v.z, s.z, h.z); v.w = fmaf(v.w, s.w, h.w);
    if (p.pre_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
  }
  return v;
}

// Fused epilogue for one output element (row m, column n); urow = per-utterance(/segment) row for ubias & gate.
__device__ __forceinline__ float epilogue1(const ConvParams& p, float acc, int m, int n, int urow) {
  float v = acc;
  if (p.bias) v += __ldg(p.bias + n);
  if (p.ubias) v += __ldg(p.ubias + (size_t)urow * p.N + n);
  v = apply_act(v, p.act);
  if (p.post_s) v = fmaf(v, __ldg(p.post_s + n), __ldg(p.post_h + n));
  if (p.gate) v *= __ldg(p.gate + (size_t)urow * p.N + n);
  if (p.res) v += __ldg(p.res + (size_t)m * p.res_ld + p.res_coff + n);
  return apply_act(v, p.act2);
}

// Optional accumulate-into view: sum[m, n] += y (each element is owned by exactly one thread of one launch).
__device__ __forceinline__ void sum_add1(const ConvParams& p, int m, int n, float y) {
  if (p.sum) p.sum[(size_t)m * p.sum_ld + p.sum_coff + n] += y;
}
__device__ __forceinline__ void sum_add4(const ConvParams& p, int m, int n, float4 y) {
  if (p.sum) {
    float4* q = reinterpret_cast<float4*>(p.sum + (size_t)m * p.sum_ld + p.sum_coff + n);
    float4 s = *q;
    s.x += y.x; s.y += y.y; s.z += y.z; s.w += y.w;
    *q = s;
  }
}

__device__ __forceinline__ int urow_of(const ConvParams& p, int m) {
  int per = p.Tout * p.Fout;
  int b = m / per;
  int to = (m - b * per) / p.Fout;
  int s = to / p.seg_len;
  if (s >= p.n_seg) s = p.n_seg - 1;
  return b * p.n_seg + s;
}

}  // namespace vpb
