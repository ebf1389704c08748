// C ABI (include/vpb200.h): handle / weight arena / front-end state / program validation + straight-line executor.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "kernels.cuh"


using namespace vpb;

struct vp_handle {
  int device = 0;
  std::string err;
  // weights
  float* d_weights = nullptr;
  size_t weights_bytes = 0;
  // bumped by every vp_weights_load, failed or not: a program validated against an older blob (its weight offsets and
  // extents, its fp16 images' descale) must not run against the new one, nor its graph read the freed allocation
  int weights_gen = 0;
  // ONE workspace arena shared by all programs of the handle (a handle runs one program at a time, stream-ordered):
  // sized to the largest live program, so serving ragged lengths costs max(ws), not sum(ws), of device memory
  char* d_arena = nullptr;
  size_t arena_bytes = 0;
  cudaStream_t cap_stream = nullptr;   // private stream CUDA graphs are captured on (the caller's may be the legacy default)
  // front-end
  bool fe_set = false;
  vp_frontend_desc fe{};
  vp_frontend_options fe_opt{VP_FRAME_DEFAULT, 0, 1.0};
  float* d_window = nullptr;
  double2* d_twiddle = nullptr;
  int* d_mel_start = nullptr;
  int* d_mel_count = nullptr;
  int* d_mel_off = nullptr;
  double* d_mel_w = nullptr;   // the bank's weights widened to fp64, as the mel accumulation consumes them
  int mel_nw = 0;
  float* d_dct = nullptr;
  HfState* hf = nullptr;       // the HF wav2vec 2.0 / WavLM front-end (vp_frontend_set_hf) instead of the above
};

struct vp_program {
  vp_handle* h = nullptr;
  std::vector<vp_op> ops;
  std::vector<int> engines;   // resolved conv engine per op (VP_ENGINE_FFMA / VP_ENGINE_TC), 0 for non-conv
  // fused Res2Net chains (res2_chain_len): chain[i] = n > 1 at the first op of a chain of n ops launched as one
  // res2_chain_kernel, -1 at the chain's other ops, 0 elsewhere
  std::vector<int> chain;
  size_t ws_bytes = 0, in_floats = 0, out_floats = 0;
  int launches = 0;
  int B = 0;                  // utterances (every op of a program agrees on it)
  // CUDA graph of one vp_embed (all ops + the slot memset), keyed on the pointers baked into its nodes
  cudaGraphExec_t gexec = nullptr;
  const float* g_feats = nullptr;
  float* g_emb = nullptr;
  char* g_arena = nullptr;
  int runs = 0, g_miss = 0;
  bool g_off = false;
  int n_slots = 0;            // amax slots (uint32 each) behind the workspace, zeroed at the start of every run
  int weights_gen = 0;        // the handle's weights_gen the program was validated against
  size_t arena_need() const { return ws_bytes + (((size_t)n_slots * 4 + 255) & ~(size_t)255); }
  unsigned* slot(int32_t q) const { return q > 0 ? reinterpret_cast<unsigned*>(h->d_arena + ws_bytes) + (q - 1) : nullptr; }
};

static int fail(vp_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  return code;
}
#define CUDA_TRY(h, expr)                                                                          \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess) return fail(h, VP_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

static const int FPB = 16;   // frames per front-end CTA

// VP_ENGINE_AUTO prefers the two-term FP16 split of the tensor-core engine where an op is eligible (conv_tc16_supported);
// VPB_TC_F16=0 keeps AUTO on split TF32, the bit-invariant reference engine.
static bool tc16_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("VPB_TC_F16"); on = (e && e[0] == '0') ? 0 : 1; }
  return on == 1;
}

extern "C" {

static void fill_conv(const vp_program* p, const vp_op& o, const float* feats, float* emb, vpb::ConvParams& c);

int vp_abi_version(void) { return VP_ABI_VERSION; }
int32_t vp_sizeof_op(void) { return (int32_t)sizeof(vp_op); }
int32_t vp_sizeof_frontend_desc(void) { return (int32_t)sizeof(vp_frontend_desc); }
int32_t vp_sizeof_frontend_options(void) { return (int32_t)sizeof(vp_frontend_options); }
int32_t vp_sizeof_hf_desc(void) { return (int32_t)sizeof(vp_hf_desc); }

int vp_create(int device, vp_handle** out) {
  if (!out) return VP_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || device < 0 || device >= n) return VP_ERR_CUDA;   // no GPU -> loud failure, no CPU path
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return VP_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return VP_ERR_UNSUPPORTED;       // sm_90a binary only
  if (cudaSetDevice(device) != cudaSuccess) return VP_ERR_CUDA;
  vp_handle* h = new (std::nothrow) vp_handle();
  if (!h) return VP_ERR_NOMEM;
  h->device = device;
  *out = h;
  return VP_OK;
}

static void free_frontend(vp_handle* h) {
  cudaFree(h->d_window); cudaFree(h->d_twiddle); cudaFree(h->d_mel_start); cudaFree(h->d_mel_count);
  cudaFree(h->d_mel_off); cudaFree(h->d_mel_w); cudaFree(h->d_dct);
  h->d_dct = nullptr;
  h->d_window = nullptr; h->d_twiddle = nullptr; h->d_mel_start = h->d_mel_count = h->d_mel_off = nullptr;
  h->d_mel_w = nullptr;
  hf_destroy(h->hf);
  h->hf = nullptr;
  h->fe_set = false;
}

void vp_destroy(vp_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  free_frontend(h);
  cudaFree(h->d_weights);
  cudaFree(h->d_arena);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  delete h;
}

const char* vp_last_error(const vp_handle* h) { return h ? h->err.c_str() : "null handle"; }

int vp_frontend_set(vp_handle* h, const vp_frontend_desc* d, const float* window, const int32_t* mel_start,
                    const int32_t* mel_count, const int32_t* mel_off, const float* mel_w, int32_t n_w, const float* dct) {
  if (!h || !d || !window || !mel_start || !mel_count || !mel_off || !mel_w) return fail(h, VP_ERR_INVALID, "null argument");
  const int N = d->n_fft;
  int rem = N > 0 ? N : 1;
  for (int f : {2, 3, 5}) while (rem % f == 0) rem /= f;
  if (N < 64 || N > 2048 || (N & 3) || rem != 1)
    return fail(h, VP_ERR_UNSUPPORTED, "n_fft %d: need 2^a 3^b 5^c, a multiple of 4, in [64, 2048]", N);
  if (d->kind != 0 && d->kind != 1) return fail(h, VP_ERR_INVALID, "front-end kind %d", d->kind);
  if (d->win_length < 2 || d->win_length > N || d->hop < 1) return fail(h, VP_ERR_INVALID, "bad window/hop");
  if (d->kind == 1 && d->win_length != N) return fail(h, VP_ERR_INVALID, "stft framing needs a window of n_fft taps");
  if (d->n_mels < 1 || d->n_mels > N / 2 + 1) return fail(h, VP_ERR_UNSUPPORTED, "n_mels %d out of range", d->n_mels);
  if (d->power != 1 && d->power != 2) return fail(h, VP_ERR_UNSUPPORTED, "power must be 1 or 2");
  if (d->use_log < 0 || d->use_log > 3) return fail(h, VP_ERR_INVALID, "use_log %d", d->use_log);
  if (d->post != 0 && d->post != 1) return fail(h, VP_ERR_INVALID, "post %d", d->post);
  if (d->post == 1) {
    if (d->kind != 1) return fail(h, VP_ERR_UNSUPPORTED, "MFCC needs stft framing");
    if (!dct) return fail(h, VP_ERR_INVALID, "MFCC needs the DCT matrix");
    if (d->n_mels > 128 || d->n_out < 1 || d->n_out > d->n_mels)
      return fail(h, VP_ERR_UNSUPPORTED, "MFCC: n_mels %d (<= 128), n_out %d (<= n_mels)", d->n_mels, d->n_out);
  }
  for (int m = 0; m < d->n_mels; ++m) {
    if (mel_count[m] < 0 || mel_start[m] < 0 || mel_start[m] + mel_count[m] > N / 2 + 1 || mel_off[m] < 0 ||
        mel_off[m] + mel_count[m] > n_w)
      return fail(h, VP_ERR_INVALID, "mel filter %d out of range", m);
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  free_frontend(h);
  std::vector<double2> tw(N);
  for (int k = 0; k < N; ++k) {
    double a = -2.0 * M_PI * (double)k / (double)N;
    tw[k] = make_double2(cos(a), sin(a));
  }
  const int F = d->n_mels;
  CUDA_TRY(h, cudaMalloc(&h->d_window, sizeof(float) * d->win_length));
  std::vector<double2> twx(N + 8);
  frontend_twiddle_table(N, tw.data(), twx.data());
  std::vector<double> mel_wd(mel_w, mel_w + (n_w > 0 ? n_w : 0));
  CUDA_TRY(h, cudaMalloc(&h->d_twiddle, sizeof(double2) * (N + 8)));
  CUDA_TRY(h, cudaMalloc(&h->d_mel_start, sizeof(int) * F));
  CUDA_TRY(h, cudaMalloc(&h->d_mel_count, sizeof(int) * F));
  CUDA_TRY(h, cudaMalloc(&h->d_mel_off, sizeof(int) * F));
  CUDA_TRY(h, cudaMalloc(&h->d_mel_w, sizeof(double) * (n_w > 0 ? n_w : 1)));
  CUDA_TRY(h, cudaMemcpy(h->d_window, window, sizeof(float) * d->win_length, cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(h->d_twiddle, twx.data(), sizeof(double2) * (N + 8), cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(h->d_mel_start, mel_start, sizeof(int) * F, cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(h->d_mel_count, mel_count, sizeof(int) * F, cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(h->d_mel_off, mel_off, sizeof(int) * F, cudaMemcpyHostToDevice));
  if (n_w > 0) CUDA_TRY(h, cudaMemcpy(h->d_mel_w, mel_wd.data(), sizeof(double) * n_w, cudaMemcpyHostToDevice));
  h->mel_nw = n_w > 0 ? n_w : 0;
  if (d->post == 1) {
    CUDA_TRY(h, cudaMalloc(&h->d_dct, sizeof(float) * F * d->n_out));
    CUDA_TRY(h, cudaMemcpy(h->d_dct, dct, sizeof(float) * F * d->n_out, cudaMemcpyHostToDevice));
  }
  h->fe = *d;
  h->fe_opt = vp_frontend_options{VP_FRAME_DEFAULT, 0, 1.0};
  h->fe_set = true;
  return VP_OK;
}

int vp_frontend_set_hf(vp_handle* h, const vp_hf_desc* d, const float* const* conv_w, const float* const* conv_b,
                       const float* const* norm_w, const float* const* norm_b, const float* proj_w, const float* proj_b) {
  if (!h || !d || !conv_w || !proj_w || !proj_b) return fail(h, VP_ERR_INVALID, "null argument");
  const char* derr = hf_desc_error(*d);
  if (*derr) return fail(h, VP_ERR_UNSUPPORTED, "HF front-end: %s", derr);
  for (int l = 0; l < d->n_layers; ++l) {
    if (!conv_w[l] || (d->conv_bias && (!conv_b || !conv_b[l])))
      return fail(h, VP_ERR_INVALID, "HF front-end: layer %d conv weight / bias missing", l);
    if ((d->norm == VP_HF_NORM_LAYER || l == 0) && (!norm_w || !norm_b || !norm_w[l] || !norm_b[l]))
      return fail(h, VP_ERR_INVALID, "HF front-end: layer %d norm affine missing", l);
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  free_frontend(h);
  HfState* s = nullptr;
  CUDA_TRY(h, hf_create(*d, conv_w, conv_b, norm_w, norm_b, proj_w, proj_b, &s));
  h->hf = s;
  h->fe = vp_frontend_desc{};
  h->fe_opt = vp_frontend_options{VP_FRAME_DEFAULT, 0, 1.0};
  h->fe_set = true;
  return VP_OK;
}

int vp_frontend_set_options(vp_handle* h, const vp_frontend_options* o) {
  if (!h || !o) return fail(h, VP_ERR_INVALID, "null argument");
  if (!h->fe_set) return fail(h, VP_ERR_INVALID, "front-end not configured (vp_frontend_set)");
  if (h->hf) return fail(h, VP_ERR_INVALID, "the HF front-end has no framing options");
  const bool kaldi = h->fe.kind == 0;
  const int m = o->frame_mode;
  if (kaldi ? (m != VP_FRAME_DEFAULT && m != VP_FRAME_KALDI_REFLECT)
            : (m != VP_FRAME_DEFAULT && (m < VP_FRAME_STFT_CONSTANT || m > VP_FRAME_STFT_NOCENTER)))
    return fail(h, VP_ERR_INVALID, "frame mode %d does not fit front-end kind %d", m, h->fe.kind);
  if (o->pad < 0 || (kaldi && o->pad != 0)) return fail(h, VP_ERR_INVALID, "pad %d (kind 1 only, >= 0)", o->pad);
  if (!(o->spec_scale > 0.0) || !std::isfinite(o->spec_scale) || (kaldi && o->spec_scale != 1.0))
    return fail(h, VP_ERR_INVALID, "spec_scale %g (finite, > 0; 1 for kind 0)", o->spec_scale);
  h->fe_opt = *o;
  return VP_OK;
}

int32_t vp_num_frames(const vp_handle* h, int32_t n) {
  if (!h || !h->fe_set) return -1;
  if (h->hf) return hf_frames(h->hf, n);
  return frontend_frames(h->fe.kind, h->fe_opt.frame_mode, h->fe.win_length, h->fe.n_fft, h->fe.hop, h->fe_opt.pad, n);
}

// The waveform lengths torch accepts for the configured framing (kaldi.py:141, torch.stft / F.pad): "" when L fits.
static const char* frontend_length_error(const vp_handle* h, int L) {
  const int64_t Lp = (int64_t)L + 2 * (int64_t)h->fe_opt.pad, half = h->fe.n_fft / 2;
  switch (h->fe.kind == 0 ? -1 : h->fe_opt.frame_mode) {
    case -1: return (h->fe.win_length >= 2 && h->fe.win_length <= L) ? "" : "kaldi framing needs 2 <= win_length <= L";
    case VP_FRAME_DEFAULT: return half < Lp ? "" : "reflect padding needs n_fft/2 < L + 2 pad";
    case VP_FRAME_STFT_CIRCULAR: return half <= Lp ? "" : "circular padding needs n_fft/2 <= L + 2 pad";
    case VP_FRAME_STFT_NOCENTER: return h->fe.n_fft <= Lp ? "" : "center=False needs n_fft <= L + 2 pad";
    default: return L >= 1 ? "" : "empty waveform";
  }
}

int32_t vp_feature_dim(const vp_handle* h) {
  if (!h || !h->fe_set) return -1;
  if (h->hf) return hf_feature_dim(h->hf);
  return h->fe.post == 1 ? h->fe.n_out : h->fe.n_mels;
}

static size_t round4(size_t n) { return (n + 3) & ~(size_t)3; }

// scratch layout of a call with T frames: [CMN partial sums B*nblk*F], for MFCC [per-CTA maxima B*nblk] [dB mel values
// B*T*n_mels], then [the rows' frame counts: B int32] of a ragged call
static size_t frontend_scratch_floats(const vp_handle* h, int B, int T) {
  size_t nblk = (T + FPB - 1) / FPB;
  size_t n = round4((size_t)B * nblk * vp_feature_dim(h));
  if (h->fe.post == 1) n += round4((size_t)B * nblk) + round4((size_t)B * T * h->fe.n_mels);
  return n;
}
size_t vp_frontend_scratch_floats(const vp_handle* h, int32_t B, int32_t Lpad) {
  if (h && h->fe_set && h->hf) return hf_scratch_floats(h->hf, B, Lpad);
  int T = vp_num_frames(h, Lpad);
  if (T <= 0) return 0;
  return frontend_scratch_floats(h, B, T) + round4((size_t)B);
}

// The waveform length check of every front-end call: "" when B rows of L samples give at least one frame.
static const char* frontend_call_error(const vp_handle* h, int B, int L) {
  if (B < 1) return "empty batch";
  if (h->hf) return hf_frames(h->hf, L) < 1 ? "shorter than the feature encoder's receptive field" : "";
  const char* len_err = frontend_length_error(h, L);
  if (*len_err) return len_err;
  return vp_num_frames(h, L) < 1 ? "shorter than one frame" : "";
}

// The planned FrontendParams of a call on B rows of L samples (frontend_call_error(h, B, L) == ""), buffer pointers
// left null: the one place the launch shape comes from, for run_frontend and vp_frontend_plan_info alike.  T: the
// frames of the call, vp_num_frames(L) when < 0 (a ragged call passes its longest row's).
static FrontendParams frontend_params(const vp_handle* h, int B, int L, int T = -1) {
  FrontendParams p{};
  if (T < 0) T = vp_num_frames(h, L);
  p.window = h->d_window; p.twiddle = h->d_twiddle;
  p.mel_start = h->d_mel_start; p.mel_count = h->d_mel_count; p.mel_off = h->d_mel_off; p.mel_w = h->d_mel_w;
  p.mel_nw = h->mel_nw;
  p.B = B; p.L = L; p.T = T; p.kind = h->fe.kind; p.N = h->fe.n_fft; p.WL = h->fe.win_length; p.hop = h->fe.hop;
  p.F = h->fe.n_mels; p.remove_dc = h->fe.remove_dc; p.power = h->fe.power; p.use_log = h->fe.use_log;
  p.fpb = FPB; p.nblk = (T + FPB - 1) / FPB;
  p.frame = h->fe_opt.frame_mode;
  p.pad = p.kind == 0 ? p.WL / 2 - p.hop / 2 : h->fe_opt.pad;
  p.spec_mult = h->fe.power == 2 ? h->fe_opt.spec_scale * h->fe_opt.spec_scale : h->fe_opt.spec_scale;
  p.preemph = h->fe.preemph; p.log_floor = h->fe.log_floor; p.db_mult = h->fe.db_mult;
  frontend_plan(p, h->fe.post == 1);
  return p;
}

// stage: 0 = the whole front-end; 1 = MFCC mel stage only (maximum -> ext_max[0]); 2 = MFCC clamp/DCT/CMN only, clamping
// against the externally reduced maximum ext_max[0].
// lens (device int32 [B]) non-null: a ragged call of T frames, row b featurized alone on its first lens[b] samples.
static int run_frontend(vp_handle* h, const float* wave, int B, int L, const int32_t* keep, float* feats, float* scratch,
                        cudaStream_t st, int stage = 0, float* ext_max = nullptr, const int32_t* lens = nullptr,
                        int T_call = -1) {
  if (!h) return VP_ERR_INVALID;
  if (!h->fe_set) return fail(h, VP_ERR_INVALID, "front-end not configured (vp_frontend_set)");
  if (h->hf && B >= 1 && *frontend_call_error(h, B, L))     // a short row has no features to write: say why first
    return fail(h, VP_ERR_INVALID, "waveform of %d samples: %s (%d samples): Kernel size can't be greater than actual "
                "input size", L, frontend_call_error(h, B, L), hf_min_samples(h->hf));
  if ((stage != 2 && !wave) || (stage != 1 && !feats) || !scratch || B < 1) return fail(h, VP_ERR_INVALID, "null/empty argument");
  if (stage != 0 && (h->fe.post != 1 || !ext_max)) return fail(h, VP_ERR_INVALID, "two-stage calls are for the MFCC front-end");
  const char* len_err = frontend_call_error(h, B, L);
  if (*len_err) return fail(h, VP_ERR_INVALID, "waveform of %d samples: %s", L, len_err);
  if (lens && (T_call < 1 || T_call > vp_num_frames(h, L)))
    return fail(h, VP_ERR_INVALID, "T = %d frames: need 1 <= T <= %d, the frames of a %d-sample row", T_call,
                vp_num_frames(h, L), L);
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (h->hf) {
    if (stage != 0) return fail(h, VP_ERR_INVALID, "two-stage calls are for the MFCC front-end");
    CUDA_TRY(h, hf_run(h->hf, wave, B, L, lens, lens ? T_call : vp_num_frames(h, L), keep, feats, scratch, st));
    return VP_OK;
  }
  FrontendParams p = frontend_params(h, B, L, lens ? T_call : -1);
  p.wave = wave; p.feats = feats; p.partial = scratch;
  const int T = p.T;
  if (lens) {
    p.lens = lens;
    p.row_T = reinterpret_cast<int*>(scratch + frontend_scratch_floats(h, B, T));
  }
  if (h->fe.post == 1) {
    MfccParams m;
    float* cta_max = scratch + round4((size_t)B * p.nblk * h->fe.n_out);
    float* mel = cta_max + round4((size_t)B * p.nblk);
    p.feats = mel; p.partial = nullptr; p.cta_max = cta_max;
    m.mel = mel; m.cta_max = cta_max; m.dct = h->d_dct; m.feats = feats; m.partial = scratch;
    m.B = B; m.T = T; m.M = h->fe.n_mels; m.K = h->fe.n_out; m.fpb = FPB; m.nblk = p.nblk; m.n_max = B * p.nblk;
    m.top_db = h->fe.top_db;
    m.row_T = p.row_T;
    if (stage == 1) {
      CUDA_TRY(h, launch_frontend_mfcc_mel(p, ext_max, st));
    } else if (stage == 2) {
      m.cta_max = ext_max; m.n_max = 1;
      CUDA_TRY(h, launch_frontend_mfcc_finish(p, m, keep, st));
    } else {
      CUDA_TRY(h, launch_frontend_mfcc(p, m, keep, st));
    }
    return VP_OK;
  }
  CUDA_TRY(h, launch_frontend(p, keep, st));
  return VP_OK;
}

int vp_frontend_plan_info(const vp_handle* h, int32_t B, int32_t Lpad, int32_t stage, int32_t* info) {
  if (!h || !info) return VP_ERR_INVALID;
  if (!h->fe_set || stage != h->fe.post || *frontend_call_error(h, B, Lpad)) return VP_ERR_INVALID;
  if (h->hf) {
    hf_plan(h->hf, B, Lpad, info);
    return VP_OK;
  }
  const FrontendParams p = frontend_params(h, B, Lpad);
  const int inst = frontend_instantiation(p.N);
  info[0] = inst;
  info[1] = p.G;
  info[2] = p.tpc;
  info[3] = p.cache;
  info[4] = p.n_pass;
  info[5] = frontend_mel_chains(inst, p.F, p.G) ? 1 : 0;
  info[6] = p.nblk;
  info[7] = frontend_grid_x(p);
  return VP_OK;
}

int vp_features(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep, float* feats,
                float* scratch, void* stream) {
  return run_frontend(h, wave, B, Lpad, keep, feats, scratch, (cudaStream_t)stream);
}

int vp_features_each(vp_handle* h, const float* wave, int32_t B, int32_t ld, const int32_t* lens, int32_t T, float* feats,
                     float* scratch, void* stream) {
  if (!lens) return fail(h, VP_ERR_INVALID, "null argument");
  return run_frontend(h, wave, B, ld, nullptr, feats, scratch, (cudaStream_t)stream, 0, nullptr, lens, T);
}

int vp_mfcc_mel(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, float* scratch, float* max_out, void* stream) {
  return run_frontend(h, wave, B, Lpad, nullptr, nullptr, scratch, (cudaStream_t)stream, 1, max_out);
}
int vp_mfcc_finish(vp_handle* h, int32_t B, int32_t Lpad, const int32_t* keep, float* feats, float* scratch,
                   const float* max_in, void* stream) {
  return run_frontend(h, nullptr, B, Lpad, keep, feats, scratch, (cudaStream_t)stream, 2, const_cast<float*>(max_in));
}

int vp_weights_load(vp_handle* h, const void* blob, size_t nbytes) {
  if (!h || !blob || nbytes == 0 || (nbytes & 15)) return fail(h, VP_ERR_INVALID, "weights blob must be non-empty, 16 B multiple");
  CUDA_TRY(h, cudaSetDevice(h->device));
  ++h->weights_gen;           // before the old blob is freed: every existing program is stale from here, load or no load
  cudaFree(h->d_weights);
  h->d_weights = nullptr;
  h->weights_bytes = 0;
  CUDA_TRY(h, cudaMalloc(&h->d_weights, nbytes));
  CUDA_TRY(h, cudaMemcpy(h->d_weights, blob, nbytes, cudaMemcpyHostToDevice));
  h->weights_bytes = nbytes;
  return VP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// program validation: every offset/extent an op can touch is bounds-checked once here, so kernels run unchecked.
// ---------------------------------------------------------------------------------------------------------------
static bool act_ok(int a) { return a >= VP_ACT_NONE && a <= VP_ACT_GELU; }

// extent (in floats) of a strided [rows, ld] view whose last row uses columns [coff, coff + cols)
static size_t view_floats(long long rows, int ld, int coff, int cols) {
  if (rows <= 0) return 0;
  return (size_t)(rows - 1) * ld + coff + cols;
}

static int check_act_buf(vp_program* p, const char* what, int64_t off, size_t floats, bool is_dst, int opi) {
  vp_handle* h = p->h;
  if (off == VP_BUF_INPUT) {
    if (is_dst) return fail(h, VP_ERR_INVALID, "op %d: %s writes the program input", opi, what);
    if (floats > p->in_floats) return fail(h, VP_ERR_INVALID, "op %d: %s reads %zu floats > input %zu", opi, what, floats, p->in_floats);
    return VP_OK;
  }
  if (off == VP_BUF_OUTPUT) {
    if (floats > p->out_floats) return fail(h, VP_ERR_INVALID, "op %d: %s touches %zu floats > output %zu", opi, what, floats, p->out_floats);
    return VP_OK;
  }
  if (off < 0 || (off & 15)) return fail(h, VP_ERR_INVALID, "op %d: %s offset %lld invalid/misaligned", opi, what, (long long)off);
  if ((size_t)off + floats * 4 > p->ws_bytes) return fail(h, VP_ERR_INVALID, "op %d: %s [%lld, +%zu B) exceeds workspace %zu", opi, what, (long long)off, floats * 4, p->ws_bytes);
  return VP_OK;
}
static int check_w(vp_program* p, const char* what, int64_t off, size_t floats, int opi) {
  vp_handle* h = p->h;
  if (off < 0 || (off & 15)) return fail(h, VP_ERR_INVALID, "op %d: %s weight offset %lld invalid/misaligned", opi, what, (long long)off);
  if ((size_t)off + floats * 4 > h->weights_bytes) return fail(h, VP_ERR_INVALID, "op %d: %s exceeds weight arena", opi, what);
  return VP_OK;
}
#define TRY(x) do { int r__ = (x); if (r__ != VP_OK) return r__; } while (0)

static int validate_op(vp_program* p, const vp_op& o, int i) {
  vp_handle* h = p->h;
  if (o.B < 1) return fail(h, VP_ERR_INVALID, "op %d: B", i);
  if (o.amax_out < 0 || o.amax_out > 65536 || o.amax_in < 0 || o.amax_in > 65536) return fail(h, VP_ERR_INVALID, "op %d: amax slot", i);
  if (o.amax_in > 0 && o.kind != VP_OP_CONV) return fail(h, VP_ERR_INVALID, "op %d: amax_in is a CONV field", i);
  if (o.amax_out > 0 && (o.kind == VP_OP_COLSTATS || o.kind == VP_OP_ASP_POOL))
    return fail(h, VP_ERR_UNSUPPORTED, "op %d: pooling ops do not track amax", i);
  switch (o.kind) {
    case VP_OP_CONV:
    case VP_OP_CONV_C1: {
      const int cin_tot = o.Cin + (o.src2_mode == VP_SRC2_CONCAT ? o.Cin2 : 0);
      if (o.Tin < 1 || o.Fin < 1 || o.Tout < 1 || o.Fout < 1 || o.Cin < 1 || o.Cout < 1 || o.KT < 1 || o.KF < 1 ||
          o.sT < 1 || o.sF < 1 || o.dT < 1 || o.dF < 1 || o.padT < 0 || o.padF < 0)
        return fail(h, VP_ERR_INVALID, "op %d: conv geometry", i);
      if (!act_ok(o.act) || !act_ok(o.act2)) return fail(h, VP_ERR_INVALID, "op %d: activation id", i);
      if (o.seg_len < 1 || o.n_seg < 1) return fail(h, VP_ERR_INVALID, "op %d: seg_len/n_seg", i);
      // every tap of every output position must land inside the (padded) source
      const long long t_last = (long long)(o.Tout - 1) * o.sT - o.padT + (long long)(o.KT - 1) * o.dT;
      const long long f_last = (long long)(o.Fout - 1) * o.sF - o.padF + (long long)(o.KF - 1) * o.dF;
      if (o.pad_mode == VP_PAD_REFLECT) {
        if (o.padT >= o.Tin || t_last - (o.Tin - 1) >= o.Tin || o.padF != 0 || f_last >= o.Fin)
          return fail(h, VP_ERR_INVALID, "op %d: reflect padding wider than the map (Tin=%d padT=%d)", i, o.Tin, o.padT);
      } else if (o.pad_mode != VP_PAD_ZERO) {
        return fail(h, VP_ERR_INVALID, "op %d: pad_mode", i);
      }
      const long long rows_in = (long long)o.B * o.Tin * o.Fin, rows_out = (long long)o.B * o.Tout * o.Fout;
      if (rows_out > 0x7fffffffLL || rows_in > 0x7fffffffLL) return fail(h, VP_ERR_UNSUPPORTED, "op %d: > 2^31 rows", i);
      if (o.kind == VP_OP_CONV_C1) {
        if (o.Cin != 1 || o.KT > 7 || o.KF > 7 || (o.Cout & 3) || o.w_ld < o.KT * o.KF ||
            o.src2_mode != VP_SRC2_NONE || o.pre_s >= 0 || (o.out_ld & 3) || (o.out_coff & 3) || o.pad_mode != VP_PAD_ZERO)
          return fail(h, VP_ERR_UNSUPPORTED, "op %d: CONV_C1 is a <=7x7 zero-padded conv with Cin=1, Cout%%4==0", i);
        TRY(check_w(p, "w", o.w, view_floats(o.Cout, o.w_ld, 0, o.KT * o.KF), i));
      } else {
        if ((o.Cin & 3) || (cin_tot & 3) || (o.in_ld & 3) || (o.in_coff & 3) || (o.w_ld & 3))
          return fail(h, VP_ERR_UNSUPPORTED, "op %d: CONV needs Cin/in_ld/in_coff/w_ld multiples of 4", i);
        if (o.src2_mode != VP_SRC2_NONE && ((o.src2_ld & 3) || (o.src2_coff & 3)))
          return fail(h, VP_ERR_UNSUPPORTED, "op %d: src2 alignment", i);
        if (o.src2_mode == VP_SRC2_CONCAT && (o.Cin2 < 4 || (o.Cin2 & 3))) return fail(h, VP_ERR_UNSUPPORTED, "op %d: Cin2", i);
        if (o.w_ld < o.KT * o.KF * cin_tot) return fail(h, VP_ERR_INVALID, "op %d: w_ld < K", i);
        TRY(check_w(p, "w", o.w, view_floats(o.Cout, o.w_ld, 0, o.KT * o.KF * cin_tot), i));
      }
      TRY(check_act_buf(p, "src", o.src, view_floats(rows_in, o.in_ld, o.in_coff, o.Cin), false, i));
      if (o.src2_mode != VP_SRC2_NONE)
        TRY(check_act_buf(p, "src2", o.src2, view_floats(rows_in, o.src2_ld, o.src2_coff, o.src2_mode == VP_SRC2_CONCAT ? o.Cin2 : o.Cin), false, i));
      TRY(check_act_buf(p, "dst", o.dst, view_floats(rows_out, o.out_ld, o.out_coff, o.Cout), true, i));
      if (o.res != VP_BUF_NONE) TRY(check_act_buf(p, "res", o.res, view_floats(rows_out, o.res_ld, o.res_coff, o.Cout), false, i));
      if (o.sum != VP_BUF_NONE) {
        if (o.kind == VP_OP_CONV_C1 || o.sum < 0 || (o.sum_ld & 3) || (o.sum_coff & 3) || (o.Cout & 3))
          return fail(h, VP_ERR_UNSUPPORTED, "op %d: sum view must be a 4-float aligned workspace view of a CONV op", i);
        TRY(check_act_buf(p, "sum", o.sum, view_floats(rows_out, o.sum_ld, o.sum_coff, o.Cout), true, i));
      }
      if (o.gate != VP_BUF_NONE) TRY(check_act_buf(p, "gate", o.gate, (size_t)o.B * o.n_seg * o.Cout, false, i));
      if (o.ubias != VP_BUF_NONE) TRY(check_act_buf(p, "ubias", o.ubias, (size_t)o.B * o.n_seg * o.Cout, false, i));
      if (o.w_tc >= 0) {
        if (o.kind != VP_OP_CONV || o.tc_bn < 16 || o.tc_bn > 256 || (o.tc_bn & 15)) return fail(h, VP_ERR_INVALID, "op %d: tc_bn", i);
        const size_t nt = (o.Cout + o.tc_bn - 1) / o.tc_bn, kb = ((size_t)o.KT * o.KF * cin_tot + 31) / 32;
        if (o.w_tc & 127) return fail(h, VP_ERR_INVALID, "op %d: w_tc must be 128 B aligned", i);
        TRY(check_w(p, "w_tc", o.w_tc, nt * kb * 2 * (size_t)o.tc_bn * 32, i));
      }
      if (o.bias >= 0) TRY(check_w(p, "bias", o.bias, o.Cout, i));
      if (o.pre_s >= 0) { TRY(check_w(p, "pre_s", o.pre_s, cin_tot, i)); TRY(check_w(p, "pre_h", o.pre_h, cin_tot, i)); }
      if (o.post_s >= 0) { TRY(check_w(p, "post_s", o.post_s, o.Cout, i)); TRY(check_w(p, "post_h", o.post_h, o.Cout, i)); }
      return VP_OK;
    }
    case VP_OP_COLSTATS: {
      const long long R = (long long)o.Tin * o.Fin;
      if (R < 1 || o.Cin < 1) return fail(h, VP_ERR_INVALID, "op %d: stats geometry", i);
      if (o.mode < VP_STATS_MEAN || o.mode > VP_STATS_MEAN_VAR_UNBIASED) return fail(h, VP_ERR_INVALID, "op %d: stats mode", i);
      if ((o.mode == VP_STATS_MEAN_STD_UNBIASED || o.mode == VP_STATS_MEAN_STD_TSTP || o.mode == VP_STATS_MEAN_VAR_UNBIASED) && R < 2)
        return fail(h, VP_ERR_INVALID, "op %d: unbiased std needs >= 2 rows", i);
      TRY(check_act_buf(p, "src", o.src, view_floats((long long)o.B * R, o.in_ld, o.in_coff, o.Cin), false, i));
      if (o.mode == VP_STATS_SEG_CONTEXT) {
        if (o.seg_len < 1 || o.n_seg != (int)((R + o.seg_len - 1) / o.seg_len))
          return fail(h, VP_ERR_INVALID, "op %d: n_seg must be ceil(R/seg_len)", i);
        TRY(check_act_buf(p, "dst", o.dst, view_floats((long long)o.B * o.n_seg, o.out_ld, o.out_coff, o.Cin), true, i));
      } else {
        const int cols = o.mode == VP_STATS_MEAN ? o.Cin : 2 * o.Cin;
        TRY(check_act_buf(p, "dst", o.dst, view_floats(o.B, o.out_ld, o.out_coff, cols), true, i));
      }
      return VP_OK;
    }
    case VP_OP_ASP_POOL: {
      if (o.Tin < 1 || o.Cin < 1) return fail(h, VP_ERR_INVALID, "op %d: asp geometry", i);
      const long long rows = (long long)o.B * o.Tin;
      TRY(check_act_buf(p, "x", o.src, view_floats(rows, o.in_ld, o.in_coff, o.Cin), false, i));
      TRY(check_act_buf(p, "logits", o.src2, view_floats(rows, o.src2_ld, o.src2_coff, o.Cin), false, i));
      if (o.mode != 0 && o.mode != 1) return fail(h, VP_ERR_INVALID, "op %d: asp mode", i);
      TRY(check_act_buf(p, "dst", o.dst, view_floats(o.B, o.out_ld, o.out_coff, (o.mode == 1 ? 1 : 2) * o.Cin), true, i));
      return VP_OK;
    }
    case VP_OP_POOL2D: {
      if (o.Tin < 1 || o.Fin < 1 || o.Tout < 1 || o.Fout < 1 || o.KT < 1 || o.KF < 1 || o.sT < 1 || o.sF < 1 || o.padT < 0 ||
          o.padF < 0 || o.Cin < 4 || (o.Cin & 3) || (o.in_ld & 3) || (o.in_coff & 3) || (o.out_ld & 3) || (o.out_coff & 3) ||
          (o.mode != 0 && o.mode != 1))
        return fail(h, VP_ERR_INVALID, "op %d: pool geometry / alignment", i);
      if ((long long)(o.Tout - 1) * o.sT - o.padT >= o.Tin || (long long)(o.Fout - 1) * o.sF - o.padF >= o.Fin ||
          o.padT >= o.KT || o.padF >= o.KF)
        return fail(h, VP_ERR_INVALID, "op %d: pooling window entirely outside the map", i);
      TRY(check_act_buf(p, "src", o.src, view_floats((long long)o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin), false, i));
      TRY(check_act_buf(p, "dst", o.dst, view_floats((long long)o.B * o.Tout * o.Fout, o.out_ld, o.out_coff, o.Cin), true, i));
      return VP_OK;
    }
    case VP_OP_EW: {
      const long long rows = (long long)o.B * o.Tin * o.Fin;
      if (o.mode == VP_EW_PAD_COPY) {
        if (rows < 1 || o.Cin < 1 || o.Cout < o.Cin || (o.Cout & 3) || (o.out_ld & 3) || (o.out_coff & 3))
          return fail(h, VP_ERR_UNSUPPORTED, "op %d: PAD_COPY shape", i);
        TRY(check_act_buf(p, "x", o.src, view_floats(rows, o.in_ld, o.in_coff, o.Cin), false, i));
        TRY(check_act_buf(p, "dst", o.dst, view_floats(rows, o.out_ld, o.out_coff, o.Cout), true, i));
        return VP_OK;
      }
      if (rows < 1 || o.Cin < 4 || (o.Cin & 3) || (o.in_ld & 3) || (o.in_coff & 3) || (o.out_ld & 3) || (o.out_coff & 3))
        return fail(h, VP_ERR_UNSUPPORTED, "op %d: EW alignment", i);
      if (!act_ok(o.act2)) return fail(h, VP_ERR_INVALID, "op %d: activation id", i);
      TRY(check_act_buf(p, "x", o.src, view_floats(rows, o.in_ld, o.in_coff, o.Cin), false, i));
      TRY(check_act_buf(p, "dst", o.dst, view_floats(rows, o.out_ld, o.out_coff, o.Cin), true, i));
      if (o.mode == VP_EW_GATE_RES) {
        if (o.gate != VP_BUF_NONE) TRY(check_act_buf(p, "gate", o.gate, (size_t)o.B * o.Cin, false, i));
        if (o.res != VP_BUF_NONE) {
          if ((o.res_ld & 3) || (o.res_coff & 3)) return fail(h, VP_ERR_UNSUPPORTED, "op %d: res alignment", i);
          TRY(check_act_buf(p, "res", o.res, view_floats(rows, o.res_ld, o.res_coff, o.Cin), false, i));
        }
      } else if (o.mode == VP_EW_AFF) {
        if ((o.src2_ld & 3) || (o.src2_coff & 3) || (o.res_ld & 3) || (o.res_coff & 3)) return fail(h, VP_ERR_UNSUPPORTED, "op %d: AFF alignment", i);
        TRY(check_act_buf(p, "y", o.src2, view_floats(rows, o.src2_ld, o.src2_coff, o.Cin), false, i));
        TRY(check_act_buf(p, "att", o.res, view_floats(rows, o.res_ld, o.res_coff, o.Cin), false, i));
      } else if (o.mode != VP_EW_COPY) {
        return fail(h, VP_ERR_INVALID, "op %d: EW mode", i);
      }
      return VP_OK;
    }
    default:
      return fail(h, VP_ERR_INVALID, "op %d: unknown kind %d", i, o.kind);
  }
}

// A Res2Net chain op of the fused kernel: a tensor-core k3 reflect conv of width w = Cin = Cout (a multiple of 16, at most
// 64) over frames, stride 1, pad = dilation, with the simple epilogue (bias, ReLU, post affine) and no fp16 scale input.
static bool res2_op_ok(const vp_program* p, int i) {
  const vp_op& o = p->ops[i];
  if (o.kind != VP_OP_CONV || p->engines[i] != VP_ENGINE_TC) return false;
  if (o.Fin != 1 || o.Fout != 1 || o.Tin != o.Tout || o.KT != 3 || o.KF != 1 || o.sT != 1 || o.sF != 1) return false;
  if (o.pad_mode != VP_PAD_REFLECT || o.padT != o.dT || o.padF != 0) return false;
  if (o.Cin != o.Cout || o.tc_bn != o.Cout || !res2_chain_supported(o.Cout, o.Tout, o.dT)) return false;
  if (o.src2_mode == VP_SRC2_CONCAT || o.pre_s >= 0 || o.tc_kc != 0 || o.amax_in != 0) return false;
  if (o.res != VP_BUF_NONE || o.gate != VP_BUF_NONE || o.ubias != VP_BUF_NONE || o.sum != VP_BUF_NONE) return false;
  return (o.act == VP_ACT_NONE || o.act == VP_ACT_RELU) && o.act2 == VP_ACT_NONE;
}

// Length of the Res2Net chain starting at op i (0 when fewer than two ops): consecutive res2_op_ok ops of one geometry
// and one activation (the kernel applies op 0's to every op),
// op k reading column window k of one source tensor and writing window k of one destination tensor, every op after the
// first adding the previous op's output (SRC2_ADD), one amax slot, and source and destination apart in memory.
static int res2_chain_len(const vp_program* p, int i) {
  const int n_ops = (int)p->ops.size();
  if (!res2_op_ok(p, i) || p->ops[i].src2_mode != VP_SRC2_NONE) return 0;
  const vp_op& f = p->ops[i];
  const int w = f.Cout;
  int n = 1;
  while (n < RES2_MAX_OPS && i + n < n_ops && res2_op_ok(p, i + n)) {
    const vp_op& o = p->ops[i + n];
    const vp_op& q = p->ops[i + n - 1];
    if (o.B != f.B || o.Tout != f.Tout || o.dT != f.dT || o.Cout != w || o.act != f.act || o.amax_out != f.amax_out) break;
    if (o.src != f.src || o.in_ld != f.in_ld || o.in_coff != q.in_coff + w) break;
    if (o.dst != f.dst || o.out_ld != f.out_ld || o.out_coff != q.out_coff + w) break;
    if (o.src2_mode != VP_SRC2_ADD || o.src2 != q.dst || o.src2_ld != q.out_ld || o.src2_coff != q.out_coff) break;
    ++n;
  }
  if (n < 2) return 0;
  // the kernel reads op k + 1's source while it writes op k's output: the two views must not share a byte
  const long long rows = (long long)f.B * f.Tout;
  const int64_t s0 = f.src + 4 * (int64_t)f.in_coff, s1 = f.src + 4 * (int64_t)view_floats(rows, f.in_ld, f.in_coff + (n - 1) * w, w);
  const int64_t d0 = f.dst + 4 * (int64_t)f.out_coff, d1 = f.dst + 4 * (int64_t)view_floats(rows, f.out_ld, f.out_coff + (n - 1) * w, w);
  const bool src_ws = f.src >= 0, dst_ws = f.dst >= 0;
  if (src_ws == dst_ws && (src_ws || f.src == f.dst) && s0 < d1 && d0 < s1) return 0;
  return n;
}

int vp_program_create(vp_handle* h, const vp_op* ops, int32_t n_ops, size_t ws_bytes, size_t in_floats,
                      size_t out_floats, vp_program** out) {
  if (!h || !ops || n_ops < 1 || !out) return fail(h, VP_ERR_INVALID, "null/empty program");
  if (!h->d_weights) return fail(h, VP_ERR_INVALID, "load weights before creating a program");
  *out = nullptr;
  vp_program* p = new (std::nothrow) vp_program();
  if (!p) return fail(h, VP_ERR_NOMEM, "host alloc");
  p->h = h;
  p->weights_gen = h->weights_gen;
  p->ops.assign(ops, ops + n_ops);
  p->ws_bytes = (ws_bytes + 255) & ~(size_t)255;
  p->in_floats = in_floats;
  p->out_floats = out_floats;
  p->B = p->ops[0].B;
  for (int i = 0; i < n_ops; ++i)
    if (p->ops[i].src == VP_BUF_INPUT) { p->B = p->ops[i].B; break; }      // utterances of the op that reads the features
  for (int i = 0; i < n_ops; ++i) {
    int r = validate_op(p, p->ops[i], i);
    if (r != VP_OK) { delete p; return r; }
  }
  p->launches = n_ops;
  p->engines.assign(n_ops, 0);
  for (int i = 0; i < n_ops; ++i) {
    const vp_op& o = p->ops[i];
    if (o.amax_out > p->n_slots) p->n_slots = o.amax_out;
    if (o.amax_in > p->n_slots) p->n_slots = o.amax_in;
  }
  if (p->n_slots > 0) ++p->launches;             // the memset node that zeroes the slots
  for (int i = 0; i < n_ops; ++i) {
    const vp_op& o = p->ops[i];
    if (o.kind != VP_OP_CONV) continue;
    ConvParams c;
    fill_conv(p, o, nullptr, nullptr, c);
    c.amax_in = o.amax_in > 0 ? reinterpret_cast<const unsigned*>(8) : nullptr;     // eligibility only (not dereferenced)
    const bool ok = conv_tc_supported(c);
    bool ok16 = ok && o.w_tc16_q > 0 && o.tc16_descale > 0.f && conv_tc16_supported(c);
    if (ok16) {
      const int bn = o.tc_bn, nt = (o.Cout + bn - 1) / bn, kb = (c.K + 63) / 64;
      const size_t off = (size_t)(o.w_tc16_q - 1) << 4, bytes = (size_t)nt * kb * 2 * bn * 128;
      if (off + bytes > h->weights_bytes) {
        int r = fail(h, VP_ERR_INVALID, "op %d: fp16 weight image out of range", i);
        delete p;
        return r;
      }
    }
    if ((o.engine == VP_ENGINE_TC && !ok) || (o.engine == VP_ENGINE_TC16 && !ok16)) {
      int r = fail(h, VP_ERR_UNSUPPORTED, "op %d: shape / operands not supported by the requested tensor-core engine", i);
      delete p;
      return r;
    }
    if (o.engine == VP_ENGINE_TC16 || (o.engine == VP_ENGINE_AUTO && ok16 && tc16_enabled())) p->engines[i] = VP_ENGINE_TC16;
    else if (o.engine == VP_ENGINE_TC || (o.engine == VP_ENGINE_AUTO && ok)) p->engines[i] = VP_ENGINE_TC;
    else p->engines[i] = VP_ENGINE_FFMA;
  }
  p->chain.assign(n_ops, 0);
  for (int i = 0; i < n_ops;) {
    const int n = res2_chain_len(p, i);
    if (n < 2) { ++i; continue; }
    p->chain[i] = n;
    for (int k = 1; k < n; ++k) p->chain[i + k] = -1;
    p->launches -= n - 1;
    i += n;
  }
  if (cudaSetDevice(h->device) != cudaSuccess) { delete p; return fail(h, VP_ERR_CUDA, "cudaSetDevice"); }
  if (p->arena_need() > h->arena_bytes) {
    // grow the shared arena: programs enqueued earlier may still be reading the old one -> drain the device first
    const size_t want = p->arena_need() + (p->arena_need() >> 3);  // 12.5 % headroom: fewer regrows under ragged lengths
    cudaDeviceSynchronize();
    cudaFree(h->d_arena);
    h->d_arena = nullptr;
    h->arena_bytes = 0;
    if (cudaMalloc(&h->d_arena, want) != cudaSuccess) {
      cudaGetLastError();
      if (cudaMalloc(&h->d_arena, p->arena_need()) != cudaSuccess) {
        delete p;
        return fail(h, VP_ERR_NOMEM, "workspace of %zu bytes: %s", ws_bytes, cudaGetErrorString(cudaGetLastError()));
      }
      h->arena_bytes = p->arena_need();
    } else {
      h->arena_bytes = want;
    }
  }
  *out = p;
  return VP_OK;
}

void vp_program_destroy(vp_program* p) {
  if (!p) return;
  if (p->gexec) cudaGraphExecDestroy(p->gexec);
  delete p;                   // host state only: the workspace is the handle's shared arena
}

size_t vp_workspace_bytes(const vp_handle* h) { return h ? h->arena_bytes : 0; }

int32_t vp_program_launches(const vp_program* p) { return p ? p->launches : -1; }

static inline const float* rd(const vp_program* p, int64_t off, const float* in, const float* out) {
  if (off == VP_BUF_NONE) return nullptr;
  if (off == VP_BUF_INPUT) return in;
  if (off == VP_BUF_OUTPUT) return out;
  return reinterpret_cast<const float*>(p->h->d_arena + off);
}
static inline const float* wt(const vp_program* p, int64_t off) {
  return off < 0 ? nullptr : reinterpret_cast<const float*>(reinterpret_cast<const char*>(p->h->d_weights) + off);
}

static void fill_conv(const vp_program* p, const vp_op& o, const float* feats, float* emb, ConvParams& c) {
  c.src = rd(p, o.src, feats, emb);
  c.src2 = o.src2_mode == VP_SRC2_NONE ? nullptr : rd(p, o.src2, feats, emb);
  c.dst = const_cast<float*>(rd(p, o.dst, feats, emb));
  c.sum = const_cast<float*>(rd(p, o.sum, feats, emb)); c.sum_ld = o.sum_ld; c.sum_coff = o.sum_coff;
  c.res = rd(p, o.res, feats, emb); c.gate = rd(p, o.gate, feats, emb); c.ubias = rd(p, o.ubias, feats, emb);
  c.w = wt(p, o.w); c.w_tc = wt(p, o.w_tc); c.tc_bn = o.tc_bn; c.tc_kc = o.tc_kc; c.bias = wt(p, o.bias); c.pre_s = wt(p, o.pre_s); c.pre_h = wt(p, o.pre_h);
  c.post_s = wt(p, o.post_s); c.post_h = wt(p, o.post_h);
  c.B = o.B; c.Tin = o.Tin; c.Fin = o.Fin; c.Cin = o.Cin;
  c.CinTot = o.Cin + (o.src2_mode == VP_SRC2_CONCAT ? o.Cin2 : 0);
  c.in_ld = o.in_ld; c.in_coff = o.in_coff;
  c.src2_mode = o.src2_mode; c.src2_ld = o.src2_ld; c.src2_coff = o.src2_coff;
  c.Tout = o.Tout; c.Fout = o.Fout; c.out_ld = o.out_ld; c.out_coff = o.out_coff;
  c.res_ld = o.res_ld; c.res_coff = o.res_coff;
  c.KT = o.KT; c.KF = o.KF; c.sT = o.sT; c.sF = o.sF; c.dT = o.dT; c.dF = o.dF; c.padT = o.padT; c.padF = o.padF;
  c.pad_mode = o.pad_mode; c.w_ld = o.w_ld; c.pre_relu = o.pre_relu; c.act = o.act; c.act2 = o.act2;
  c.seg_len = o.seg_len; c.n_seg = o.n_seg;
  c.M = o.B * o.Tout * o.Fout; c.N = o.Cout; c.K = o.KT * o.KF * c.CinTot;
  c.amax_out = p->h->d_arena ? p->slot(o.amax_out) : nullptr;
  c.amax_in = p->h->d_arena ? p->slot(o.amax_in) : nullptr;
}

static int run_ops(vp_program* p, const float* feats, float* emb, cudaStream_t st, cudaEvent_t* evs) {
  vp_handle* h = p->h;                       // callers have made h->device current (launch attributes are per device)
  if (p->n_slots > 0) CUDA_TRY(h, cudaMemsetAsync(h->d_arena + p->ws_bytes, 0, (size_t)p->n_slots * 4, st));
  for (size_t i = 0; i < p->ops.size(); ++i) {
    const vp_op& o = p->ops[i];
    if (evs) CUDA_TRY(h, cudaEventRecord(evs[i], st));
    if (p->chain[i] < 0) continue;               // launched with its chain's first op
    if (p->chain[i] > 0) {
      Res2Args a{};
      a.n_ops = p->chain[i];
      for (int k = 0; k < a.n_ops; ++k) {
        ConvParams c;
        fill_conv(p, p->ops[i + k], feats, emb, c);
        a.src[k] = c.src + c.in_coff; a.dst[k] = c.dst + c.out_coff; a.w_tc[k] = c.w_tc;
        a.bias[k] = c.bias; a.post_s[k] = c.post_s; a.post_h[k] = c.post_h;
        if (k == 0) {
          a.amax_out = c.amax_out;
          a.W = c.N; a.B = c.B; a.T = c.Tout; a.d = c.dT; a.in_ld = c.in_ld; a.out_ld = c.out_ld;
          a.relu = c.act == VP_ACT_RELU;
        }
      }
      CUDA_TRY(h, launch_res2_chain(a, st));
      continue;
    }
    switch (o.kind) {
      case VP_OP_CONV:
      case VP_OP_CONV_C1: {
        ConvParams c;
        fill_conv(p, o, feats, emb, c);
        if (o.kind == VP_OP_CONV_C1) {
          CUDA_TRY(h, launch_conv_c1(c, st));
        } else {
          if (p->engines[i] == VP_ENGINE_TC16)
            CUDA_TRY(h, launch_conv_tc16(c, reinterpret_cast<const float*>(reinterpret_cast<const char*>(h->d_weights) + ((size_t)(o.w_tc16_q - 1) << 4)),
                                         o.tc16_descale, st));
          else if (p->engines[i] == VP_ENGINE_TC) CUDA_TRY(h, launch_conv_tc(c, st));
          else CUDA_TRY(h, launch_conv_ffma(c, st));
        }
        break;
      }
      case VP_OP_COLSTATS: {
        StatsParams s;
        s.src = rd(p, o.src, feats, emb); s.dst = const_cast<float*>(rd(p, o.dst, feats, emb));
        s.B = o.B; s.R = o.Tin * o.Fin; s.C = o.Cin; s.in_ld = o.in_ld; s.in_coff = o.in_coff;
        s.out_ld = o.out_ld; s.out_coff = o.out_coff; s.mode = o.mode; s.seg_len = o.seg_len; s.n_seg = o.n_seg;
        s.eps = o.eps;
        CUDA_TRY(h, launch_colstats(s, st));
        break;
      }
      case VP_OP_ASP_POOL: {
        AspParams a;
        a.x = rd(p, o.src, feats, emb); a.logit = rd(p, o.src2, feats, emb);
        a.dst = const_cast<float*>(rd(p, o.dst, feats, emb));
        a.B = o.B; a.T = o.Tin; a.C = o.Cin; a.x_ld = o.in_ld; a.x_coff = o.in_coff; a.l_ld = o.src2_ld;
        a.l_coff = o.src2_coff; a.out_ld = o.out_ld; a.out_coff = o.out_coff; a.eps = o.eps; a.mean_only = o.mode == 1;
        CUDA_TRY(h, launch_asp_pool(a, st));
        break;
      }
      case VP_OP_POOL2D: {
        PoolParams q;
        q.src = rd(p, o.src, feats, emb); q.dst = const_cast<float*>(rd(p, o.dst, feats, emb));
        q.B = o.B; q.Tin = o.Tin; q.Fin = o.Fin; q.Tout = o.Tout; q.Fout = o.Fout; q.C = o.Cin;
        q.in_ld = o.in_ld; q.in_coff = o.in_coff; q.out_ld = o.out_ld; q.out_coff = o.out_coff;
        q.KT = o.KT; q.KF = o.KF; q.sT = o.sT; q.sF = o.sF; q.padT = o.padT; q.padF = o.padF; q.mode = o.mode;
        q.amax_out = p->slot(o.amax_out);
        CUDA_TRY(h, launch_pool2d(q, st));
        break;
      }
      case VP_OP_EW: {
        EwParams e;
        e.x = rd(p, o.src, feats, emb);
        e.y = o.mode == VP_EW_AFF ? rd(p, o.src2, feats, emb) : nullptr;
        e.att = o.mode == VP_EW_AFF ? rd(p, o.res, feats, emb) : nullptr;
        e.gate = o.mode == VP_EW_GATE_RES ? rd(p, o.gate, feats, emb) : nullptr;
        e.res = o.mode == VP_EW_GATE_RES ? rd(p, o.res, feats, emb) : nullptr;
        e.dst = const_cast<float*>(rd(p, o.dst, feats, emb));
        e.rows = (long long)o.B * o.Tin * o.Fin; e.C = o.Cin; e.rows_per_utt = o.Tin * o.Fin;
        e.x_ld = o.in_ld; e.x_coff = o.in_coff; e.y_ld = o.src2_ld; e.y_coff = o.src2_coff;
        e.att_ld = o.res_ld; e.att_coff = o.res_coff; e.res_ld = o.res_ld; e.res_coff = o.res_coff;
        e.out_ld = o.out_ld; e.out_coff = o.out_coff; e.mode = o.mode; e.act2 = o.act2; e.C_out = o.Cout;
        e.amax_out = p->slot(o.amax_out);
        CUDA_TRY(h, launch_ew(e, st));
        break;
      }
      default:
        return fail(h, VP_ERR_INVALID, "op %zu: unknown kind", i);
    }
  }
  if (evs) CUDA_TRY(h, cudaEventRecord(evs[p->ops.size()], st));
  return VP_OK;
}

// One vp_embed = one cudaGraphLaunch: the program's launches (tens for the TDNNs, hundreds for CAM++ / the 2-D nets) are
// captured once per (feats, emb, arena) pointer triple on the handle's private stream -- the programmatic (PDL) edges
// between the kernels are kept by the capture -- and replayed on the caller's stream.  The first run of a program is
// always eager (it configures per-kernel attributes, which must not happen inside a capture).
static int embed_graph(vp_program* p, const float* feats, float* emb, cudaStream_t st) {
  vp_handle* h = p->h;
  if (!p->gexec || p->g_feats != feats || p->g_emb != emb || p->g_arena != h->d_arena) {
    if (p->gexec && ++p->g_miss > 16) {            // a caller that never reuses its buffers gains nothing from re-capturing
      p->g_off = true;
      return run_ops(p, feats, emb, st, nullptr);
    }
    if (!h->cap_stream && cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess) {
      cudaGetLastError();
      p->g_off = true;
      return run_ops(p, feats, emb, st, nullptr);
    }
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
      cudaGetLastError();
      p->g_off = true;
      return run_ops(p, feats, emb, st, nullptr);
    }
    const int r = run_ops(p, feats, emb, h->cap_stream, nullptr);
    const cudaError_t ce = cudaStreamEndCapture(h->cap_stream, &graph);
    cudaGraphExec_t ge = nullptr;
    if (r != VP_OK || ce != cudaSuccess || !graph || cudaGraphInstantiate(&ge, graph, 0) != cudaSuccess) {
      cudaGetLastError();
      if (graph) cudaGraphDestroy(graph);
      p->g_off = true;                            // this program stays on plain stream launches
      return run_ops(p, feats, emb, st, nullptr);
    }
    cudaGraphDestroy(graph);
    if (p->gexec) cudaGraphExecDestroy(p->gexec);
    p->gexec = ge;
    p->g_feats = feats; p->g_emb = emb; p->g_arena = h->d_arena;
  }
  CUDA_TRY(h, cudaGraphLaunch(p->gexec, st));
  return VP_OK;
}

// A program is lowered and validated against one weights blob; after vp_weights_load it is refused, not re-captured: its
// offsets, extents and fp16 descales belong to the old blob.
static int check_weights_gen(const vp_program* p) {
  if (p->weights_gen == p->h->weights_gen) return VP_OK;
  return fail(p->h, VP_ERR_INVALID, "program was created before the weights were reloaded: create it again");
}

int vp_embed(vp_program* p, const float* feats, float* emb, void* stream) {
  if (!p || !feats || !emb) return p ? fail(p->h, VP_ERR_INVALID, "null argument") : VP_ERR_INVALID;
  TRY(check_weights_gen(p));
  CUDA_TRY(p->h, cudaSetDevice(p->h->device));
  if (p->g_off || p->runs++ == 0) return run_ops(p, feats, emb, (cudaStream_t)stream, nullptr);
  return embed_graph(p, feats, emb, (cudaStream_t)stream);
}

int vp_embed_profiled(vp_program* p, const float* feats, float* emb, void* stream, float* ms_per_op) {
  if (!p || !feats || !emb || !ms_per_op) return p ? fail(p->h, VP_ERR_INVALID, "null argument") : VP_ERR_INVALID;
  TRY(check_weights_gen(p));
  vp_handle* h = p->h;
  const size_t n = p->ops.size();
  std::vector<cudaEvent_t> evs(n + 1);
  CUDA_TRY(h, cudaSetDevice(h->device));
  for (auto& e : evs) CUDA_TRY(h, cudaEventCreate(&e));
  int r = run_ops(p, feats, emb, (cudaStream_t)stream, evs.data());
  if (r == VP_OK) {
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) r = fail(h, VP_ERR_CUDA, "sync: %s", cudaGetErrorString(e));
  }
  if (r == VP_OK)
    for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms_per_op[i], evs[i], evs[i + 1]);
  for (auto& e : evs) cudaEventDestroy(e);
  return r;
}

int vp_program_op_info(const vp_program* p, int32_t i, int32_t* kind, int64_t* M, int64_t* N, int64_t* K, int32_t* engine) {
  if (!p || i < 0 || (size_t)i >= p->ops.size()) return VP_ERR_INVALID;
  const vp_op& o = p->ops[i];
  *kind = o.kind;
  *engine = 0;
  if (o.kind == VP_OP_CONV || o.kind == VP_OP_CONV_C1) {
    *M = (int64_t)o.B * o.Tout * o.Fout;
    *N = o.Cout;
    *K = (int64_t)o.KT * o.KF * (o.Cin + (o.src2_mode == VP_SRC2_CONCAT ? o.Cin2 : 0));
    *engine = p->engines[i];
  } else {
    *M = (int64_t)o.B * o.Tin * o.Fin; *N = o.Cin; *K = 0;
  }
  return VP_OK;
}

int vp_device_zero(void* device_ptr, size_t nbytes, void* stream) {
  if (!device_ptr) return VP_ERR_INVALID;
  return cudaMemsetAsync(device_ptr, 0, nbytes, (cudaStream_t)stream) == cudaSuccess ? VP_OK : VP_ERR_CUDA;
}

int vp_cosine_scores(vp_handle* h, const float* a, int32_t n, const float* b, int32_t m, int32_t D, float* scores, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (!a || !b || !scores || n < 1 || m < 1 || D < 1) return fail(h, VP_ERR_INVALID, "null/empty argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_cosine_scores(a, b, scores, n, m, D, (cudaStream_t)stream));
  return VP_OK;
}

size_t vp_spectral_scratch_bytes(const vp_handle* h, int32_t n) {
  (void)h;
  return n < 1 ? 0 : spectral_scratch_bytes(n);
}

int vp_spectral_laplacian(vp_handle* h, const float* emb, int32_t n, int32_t D, int32_t n_drop, double* L, void* scratch,
                          void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (!emb || !L || !scratch || n < 1 || D < 1) return fail(h, VP_ERR_INVALID, "null/empty argument");
  if (n_drop < 0 || n_drop >= n) return fail(h, VP_ERR_INVALID, "n_drop %d outside [0, n = %d)", n_drop, n);
  if ((size_t)n * sizeof(unsigned) > 227 * 1024)
    return fail(h, VP_ERR_UNSUPPORTED, "n = %d: a row of the affinity no longer fits in shared memory", n);
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_spectral_laplacian(emb, n, D, n_drop, L, scratch, (cudaStream_t)stream));
  return VP_OK;
}

int vp_sym_tridiag(vp_handle* h, double* A, int32_t n, double* d, double* e, double* tau, void* scratch, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (!A || !d || !scratch || n < 1 || (n > 1 && (!e || !tau))) return fail(h, VP_ERR_INVALID, "null/empty argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_sym_tridiag(A, n, d, e, tau, scratch, (cudaStream_t)stream));
  return VP_OK;
}

int vp_sym_tridiag_apply_q(vp_handle* h, const double* A, const double* tau, int32_t n, double* Z, int32_t k, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (!A || !Z || n < 1 || (n > 1 && !tau)) return fail(h, VP_ERR_INVALID, "null/empty argument");
  if (k < 1 || k > n || k > 16) return fail(h, VP_ERR_INVALID, "k = %d outside [1, min(n, 16)] (n = %d)", k, n);
  if ((n + 7) / 8 > apply_q_max_rows(k))
    return fail(h, VP_ERR_UNSUPPORTED, "n = %d, k = %d: the [n, k] block does not fit in the shared memory of 8 CTAs", n, k);
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_sym_tridiag_apply_q(A, tau, n, Z, k, (cudaStream_t)stream));
  return VP_OK;
}

int32_t vp_spectral_launches(int32_t n) { return n < 1 ? 0 : spectral_launches_laplacian() + spectral_launches_tridiag(n) + 1; }

size_t vp_verify_scratch_bytes(const vp_handle* h, int64_t n) {
  (void)h;
  return n < 0 || n > ((int64_t)1 << 31) ? 0 : verify_scratch_bytes(n);
}

int vp_verify_metrics(vp_handle* h, const float* scores, int64_t n, const int32_t* labels, const int32_t* trial_labels,
                      int64_t n_trials, const int32_t* enroll_labels, int64_t n_enroll, double p_target, double c_miss,
                      double c_fa, void* scratch, float* sorted_scores, uint8_t* sorted_labels, vp_verify_result* result,
                      void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (!result || !scratch || (n > 0 && !scores)) return fail(h, VP_ERR_INVALID, "null argument");
  if (n < 0 || n > ((int64_t)1 << 31)) return fail(h, VP_ERR_UNSUPPORTED, "n = %lld outside [0, 2^31]", (long long)n);
  const bool flat = labels != nullptr, matrix = trial_labels != nullptr || enroll_labels != nullptr;
  if (flat == matrix) return fail(h, VP_ERR_INVALID, "pass either labels or trial_labels + enroll_labels");
  if (matrix) {
    if (!trial_labels || !enroll_labels || n_trials < 0 || n_enroll < 0)
      return fail(h, VP_ERR_INVALID, "matrix form needs trial_labels and enroll_labels");
    if (n_trials * n_enroll != n)
      return fail(h, VP_ERR_INVALID, "n = %lld != n_trials * n_enroll = %lld * %lld", (long long)n, (long long)n_trials,
                  (long long)n_enroll);
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (n > 0)
    CUDA_TRY(h, launch_verify_sort(scores, labels, trial_labels, enroll_labels, n_enroll, n, scratch, (cudaStream_t)stream));
  CUDA_TRY(h, launch_verify_curve(n, p_target, c_miss, c_fa, scratch, sorted_scores, sorted_labels, result,
                                  (cudaStream_t)stream));
  return VP_OK;
}

int vp_resample(vp_handle* h, const float* in, int64_t in_ld, float* out, int64_t out_ld, int32_t B, const int64_t* n_in,
                const int64_t* n_out, const int32_t* up, const int32_t* down, const int64_t* tap_off, const double* taps,
                void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (B < 0 || B > 65535) return fail(h, VP_ERR_UNSUPPORTED, "B = %d outside [0, 65535]", B);
  if (B == 0 || out_ld == 0) return VP_OK;
  if (!in || !out || !n_in || !n_out || !up || !down || !tap_off || !taps || in_ld < 0 || out_ld < 0)
    return fail(h, VP_ERR_INVALID, "null argument or negative leading dimension");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_resample(in, in_ld, out, out_ld, B, n_in, n_out, up, down, tap_off, taps, (cudaStream_t)stream));
  return VP_OK;
}

size_t vp_gain_scratch_bytes(const vp_handle* h, int32_t B, int64_t ld) {
  (void)h;
  return B < 1 || ld < 0 ? 0 : gain_scratch_bytes(B, ld);
}

int vp_gain_normalize(vp_handle* h, float* wave, int64_t ld, int32_t B, const int64_t* lens, double target_db,
                      double max_gain_db, int32_t* flags, void* scratch, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (B < 0 || B > 65535) return fail(h, VP_ERR_UNSUPPORTED, "B = %d outside [0, 65535]", B);
  if (B == 0) return VP_OK;
  if (!wave || !lens || !flags || !scratch || ld < 1) return fail(h, VP_ERR_INVALID, "null/empty argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_gain(wave, ld, B, lens, target_db, max_gain_db, flags, scratch, (cudaStream_t)stream));
  return VP_OK;
}

int vp_frame_energy(vp_handle* h, const float* wave, int64_t n, int64_t hop, double* out, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (n < 0 || hop < 1 || hop > INT32_MAX) return fail(h, VP_ERR_INVALID, "n = %lld, hop = %lld: need n >= 0, 1 <= hop < 2^31",
                                                        (long long)n, (long long)hop);
  if (n / hop == 0) return VP_OK;
  if (!wave || !out) return fail(h, VP_ERR_INVALID, "null argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_frame_energy(wave, n / hop, hop, out, (cudaStream_t)stream));
  return VP_OK;
}

int vp_gather_windows(vp_handle* h, const float* src, const int64_t* offset, const int32_t* valid, int64_t n, int64_t ld,
                      float* dst, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (n < 0 || ld < 0) return fail(h, VP_ERR_INVALID, "n = %lld, ld = %lld: negative", (long long)n, (long long)ld);
  if (n == 0 || ld == 0) return VP_OK;
  if (!src || !offset || !valid || !dst) return fail(h, VP_ERR_INVALID, "null argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_gather_windows(src, offset, valid, n, ld, dst, (cudaStream_t)stream));
  return VP_OK;
}

int32_t vp_sizeof_flac_info(void) { return (int32_t)sizeof(vp_flac_info); }

size_t vp_flac_scratch_bytes(const vp_handle* h, int32_t B, int64_t nbytes, int64_t max_frames) {
  (void)h;
  return B < 1 || nbytes < 0 || max_frames < 0 ? 0 : flac_scratch_bytes(B, nbytes, max_frames);
}

int vp_flac_decode(vp_handle* h, const uint8_t* data, const int64_t* stream_off, const int64_t* frame_off,
                   const vp_flac_info* info, int32_t B, float* out, int64_t ld, int32_t* status, void* scratch,
                   int64_t nbytes, int64_t max_frames, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (B < 0 || B > 65535) return fail(h, VP_ERR_UNSUPPORTED, "B = %d outside [0, 65535]", B);
  if (B == 0) return VP_OK;
  if (nbytes < 0 || max_frames < 0 || ld < 0)
    return fail(h, VP_ERR_INVALID, "nbytes = %lld, max_frames = %lld, ld = %lld: negative", (long long)nbytes,
                (long long)max_frames, (long long)ld);
  if ((nbytes && !data) || !stream_off || !frame_off || !info || !out || !status || !scratch)
    return fail(h, VP_ERR_INVALID, "null argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_flac_decode(data, nbytes, stream_off, frame_off, info, B, max_frames, out, ld, status, scratch,
                                 (cudaStream_t)stream));
  return VP_OK;
}

int32_t vp_sizeof_pcm_info(void) { return (int32_t)sizeof(vp_pcm_info); }

int vp_pcm_decode(vp_handle* h, const uint8_t* data, int64_t nbytes, const vp_pcm_info* info, int32_t B, float* out,
                  int64_t ld, int32_t* status, void* stream) {
  if (!h) return VP_ERR_INVALID;
  if (B < 0 || B > 65535) return fail(h, VP_ERR_UNSUPPORTED, "B = %d outside [0, 65535]", B);
  if (B == 0) return VP_OK;
  if (nbytes < 0 || ld < 0)
    return fail(h, VP_ERR_INVALID, "nbytes = %lld, ld = %lld: negative", (long long)nbytes, (long long)ld);
  if ((nbytes && !data) || !info || (ld && !out) || !status) return fail(h, VP_ERR_INVALID, "null argument");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, launch_pcm_decode(data, nbytes, info, B, out, ld, status, (cudaStream_t)stream));
  return VP_OK;
}

int vp_program_peek(vp_program* p, int64_t off, size_t nbytes, void* dst, void* stream) {
  if (!p || !dst) return VP_ERR_INVALID;
  if (off < 0 || (size_t)off + nbytes > p->arena_need()) return fail(p->h, VP_ERR_INVALID, "peek out of range");
  CUDA_TRY(p->h, cudaMemcpyAsync(dst, p->h->d_arena + off, nbytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return VP_OK;
}

}  // extern "C"
