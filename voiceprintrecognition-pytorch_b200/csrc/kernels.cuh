// Kernel parameter blocks + host launchers shared between translation units.
#pragma once
#include "common.cuh"

namespace vpb {

struct FrontendParams {
  const float* wave; float* feats; float* partial;
  const float* window; const double2* twiddle;   // twiddle: the N + 8 entries of frontend_twiddle_table, in fp64
  const int* mel_start; const int* mel_count; const int* mel_off; const double* mel_w;   // weights widened to fp64
  int mel_nw;          // entries of mel_w
  int B, L, T, kind, N, WL, hop, F, remove_dc, power, use_log, fpb, nblk;
  int frame;           // VP_FRAME_* of vp_frontend_options
  int pad;             // kind 0 reflect: samples before x[0] (win/2 - hop/2, may be < 0); kind 1: torchaudio's zero pad
  double spec_mult;    // multiplies |X|^power: spec_scale^power (1.0 = none)
  float preemph, log_floor, db_mult;
  float* cta_max;      // non-null: MFCC mel stage (per-CTA maxima instead of CMN partial sums)
  int n_pass, radix[12], G;   // FFT pass plan + threads per FFT group (frontend_plan)
  int tpc, cache;             // fpb-frame tiles per CTA; 1: the CTA keeps its features in shared memory for the sums
  // Ragged call (vp_features_each): non-null lens[b] = samples of row b (L is then only the row stride); every row is
  // framed as a call of its own and its frame count T_b (frontend_frames, at most T) goes to row_T[b].
  const int* lens; int* row_T;
};
// Frames of an n-sample signal (vp_num_frames): kind 0 snip_edges / half-sample reflection, kind 1 torch.stft of the
// signal zero-extended by stft_pad at both ends, centred or not.
__host__ __device__ inline int frontend_frames(int kind, int frame, int win, int n_fft, int hop, int stft_pad, int64_t n) {
  if (kind == 0) {
    if (frame == VP_FRAME_KALDI_REFLECT) return (int)((n + hop / 2) / hop);
    return n < win ? 0 : (int)(1 + (n - win) / hop);
  }
  const int64_t Lp = n + 2 * (int64_t)stft_pad;
  if (frame == VP_FRAME_STFT_NOCENTER) return Lp < n_fft ? 0 : (int)(1 + (Lp - n_fft) / hop);
  return (int)(1 + Lp / hop);
}
// fills the line above from the shape fields (no pointer is read); mfcc_mel: the MFCC mel stage (maxima, no CMN sums)
void frontend_plan(FrontendParams& p, bool mfcc_mel);
void frontend_twiddle_table(int N, const double2* tw, double2* out);
// The launch's choices, shared by the launcher, the kernel and vp_frontend_plan_info:
// frontend_kernel<NFFT> for n_fft N (register-resident for the four power-of-two sizes, 0 = plan-driven) ...
__host__ __device__ constexpr int frontend_instantiation(int N) {
  return (N == 256 || N == 512 || N == 1024 || N == 2048) ? N : 0;
}
// ... whether its mel projection runs four interleaved chains (else the plain loop over the 2F outputs of a pair) ...
__host__ __device__ constexpr bool frontend_mel_chains(int nfft, int F, int G) { return nfft != 0 && 2 * F > G; }
// ... and its CTAs per utterance
inline int frontend_grid_x(const FrontendParams& p) { return (p.nblk + p.tpc - 1) / p.tpc; }

// MFCC tail: mel [B,T,M] dB values -> clamp(max - top_db) -> DCT [M,K] -> feats [B,T,K] + CMN partial sums.
struct MfccParams {
  const float* mel; const float* cta_max; const float* dct; float* feats; float* partial;
  int B, T, M, K, fpb, nblk, n_max;
  float top_db;        // < 0: no clamp
  const int* row_T;    // non-null: ragged call, row b has row_T[b] frames and is clamped against its own maximum
};

struct StatsParams {
  const float* src; float* dst;
  int B, R, C, in_ld, in_coff, out_ld, out_coff, mode, seg_len, n_seg;
  float eps;
};

// x: [B,T,C] view (x_ld/x_coff), logits likewise; dst[b, c] = mean, dst[b, C + c] = std.
struct AspParams {
  const float* x; const float* logit; float* dst;
  int B, T, C, x_ld, x_coff, l_ld, l_coff, out_ld, out_coff, mean_only;
  float eps;
};

struct EwParams {
  const float* x; const float* y; const float* att; const float* gate; const float* res; float* dst;
  long long rows; int C, rows_per_utt;
  int x_ld, x_coff, y_ld, y_coff, att_ld, att_coff, res_ld, res_coff, out_ld, out_coff, mode, act2;
  int C_out;   // PAD_COPY: destination width (>= C, zero filled)
  unsigned* amax_out;
};

struct PoolParams {
  const float* src; float* dst;
  int B, Tin, Fin, Tout, Fout, C, in_ld, in_coff, out_ld, out_coff, KT, KF, sT, sF, padT, padF, mode;
  unsigned* amax_out;
};
cudaError_t launch_pool2d(const PoolParams& p, cudaStream_t stream);
cudaError_t launch_cosine_scores(const float* a, const float* b, float* out, int n, int m, int D, cudaStream_t stream);

// spectral stage of the diarization clustering (spectral.cu)
size_t spectral_scratch_bytes(int n);
int spectral_launches_laplacian();
int spectral_launches_tridiag(int n);
int apply_q_max_rows(int kz);
cudaError_t launch_spectral_laplacian(const float* emb, int n, int D, int n_drop, double* L, void* scratch, cudaStream_t stream);
cudaError_t launch_sym_tridiag(double* A, int n, double* d, double* e, double* tau, void* scratch, cudaStream_t stream);
cudaError_t launch_sym_tridiag_apply_q(const double* A, const double* tau, int n, double* Z, int kz, cudaStream_t stream);

// verification metrics: stable radix sort of the scores + fp64 miss / false-alarm curves (verify.cu)
size_t verify_scratch_bytes(int64_t n);
cudaError_t launch_verify_sort(const float* scores, const int32_t* labels, const int32_t* trial, const int32_t* enroll,
                               int64_t n_enroll, int64_t n, void* scratch, cudaStream_t stream);
cudaError_t launch_verify_curve(int64_t n, double p_target, double c_miss, double c_fa, void* scratch, float* sorted_scores,
                                uint8_t* sorted_labels, vp_verify_result* result, cudaStream_t stream);

// input conditioning: polyphase resampler and dB gain (condition.cu)
cudaError_t launch_resample(const float* x, int64_t in_ld, float* y, int64_t out_ld, int B, const int64_t* n_in,
                            const int64_t* n_out, const int32_t* up, const int32_t* down, const int64_t* tap_off,
                            const double* taps, cudaStream_t stream);
size_t gain_scratch_bytes(int B, int64_t ld);
cudaError_t launch_gain(float* w, int64_t ld, int B, const int64_t* lens, double target_db, double max_gain_db,
                        int32_t* flags, void* scratch, cudaStream_t stream);

// diarization front: VAD frame energies and chunk windows of one device recording (segment.cu)
cudaError_t launch_frame_energy(const float* x, int64_t nf, int64_t hop, double* out, cudaStream_t stream);
cudaError_t launch_gather_windows(const float* src, const int64_t* offset, const int32_t* valid, int64_t rows, int64_t ld,
                                  float* dst, cudaStream_t stream);

// FLAC decoding: scan, link and decode passes over B concatenated streams (flac.cu)
size_t flac_scratch_bytes(int B, int64_t nbytes, int64_t max_frames);
cudaError_t launch_flac_decode(const uint8_t* data, int64_t nbytes, const int64_t* stream_off, const int64_t* frame_off,
                               const vp_flac_info* info, int B, int64_t max_frames, float* out, int64_t ld,
                               int32_t* status, void* scratch, cudaStream_t stream);

// PCM container samples -> float32 mono rows (pcm.cu)
cudaError_t launch_pcm_decode(const uint8_t* data, int64_t nbytes, const vp_pcm_info* info, int B, float* out,
                              int64_t ld, int32_t* status, cudaStream_t stream);

// keep: frames kept per row (the rest zeroed), or null; a ragged call (p.lens) keeps each row's own T_b instead
cudaError_t launch_frontend(const FrontendParams& p, const int* keep, cudaStream_t stream);
cudaError_t launch_frontend_mfcc(const FrontendParams& p, const MfccParams& m, const int* keep, cudaStream_t stream);
cudaError_t launch_frontend_mfcc_mel(const FrontendParams& p, float* max_out, cudaStream_t stream);
cudaError_t launch_frontend_mfcc_finish(const FrontendParams& p, const MfccParams& m, const int* keep, cudaStream_t stream);
cudaError_t launch_conv_ffma(const ConvParams& p, cudaStream_t stream);
cudaError_t launch_conv_c1(const ConvParams& p, cudaStream_t stream);
cudaError_t launch_colstats(const StatsParams& p, cudaStream_t stream);
cudaError_t launch_asp_pool(const AspParams& p, cudaStream_t stream);
cudaError_t launch_ew(const EwParams& p, cudaStream_t stream);
// tensor-core engine (conv_tc.cu, wgmma)
bool conv_tc_supported(const ConvParams& p);
cudaError_t launch_conv_tc(const ConvParams& p, cudaStream_t stream);
// two-term FP16 split of the same engine (VP_ENGINE_TC16)
bool conv_tc16_supported(const ConvParams& p);
cudaError_t launch_conv_tc16(const ConvParams& p, const float* w_tc16, float descale, cudaStream_t stream);
// fused Res2Net chain of the same engine (res2_chain_kernel): n_ops dependent k3 reflect convs of width W on one
// utterance per CTA, op j reading src[j] (+ op j-1's output) and writing dst[j]; pointers include the column offsets
constexpr int RES2_MAX_OPS = 15;
struct Res2Args {
  const float* src[RES2_MAX_OPS]; float* dst[RES2_MAX_OPS]; const float* w_tc[RES2_MAX_OPS];
  const float* bias[RES2_MAX_OPS]; const float* post_s[RES2_MAX_OPS]; const float* post_h[RES2_MAX_OPS];
  unsigned* amax_out;
  int n_ops, W, B, T, d, in_ld, out_ld, relu;
  int rows, stages;    // set by the launcher: plane rows, weight stages
};
bool res2_chain_supported(int W, int T, int d);
cudaError_t launch_res2_chain(Res2Args a, cudaStream_t stream);

// Hugging Face wav2vec 2.0 / WavLM front-end (hf.cu): the handle owns one HfState (weights packed for the tensor-core
// engine); frames, scratch and the launch sequence of a call come from here.
struct HfState;
const char* hf_desc_error(const vp_hf_desc& d);           // "" when the descriptor is one hf.cu runs
cudaError_t hf_create(const vp_hf_desc& d, const float* const* conv_w, const float* const* conv_b,
                      const float* const* norm_w, const float* const* norm_b, const float* proj_w, const float* proj_b,
                      HfState** out);
void hf_destroy(HfState* s);
int hf_frames(const HfState* s, int64_t n);
int hf_feature_dim(const HfState* s);
int hf_min_samples(const HfState* s);                     // the shortest row with one output frame
size_t hf_scratch_floats(const HfState* s, int B, int L);
void hf_plan(const HfState* s, int B, int L, int32_t* info);
// lens null: padded call (T = hf_frames(ld)); else ragged (T the longest row's frames).  keep: padded call only.
cudaError_t hf_run(const HfState* s, const float* wave, int B, int ld, const int* lens, int T, const int* keep, float* feats,
                   float* scratch, cudaStream_t st);

}  // namespace vpb
