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
};
void frontend_plan(FrontendParams& p);   // fills the line above; every other field must be set
void frontend_twiddle_table(int N, const double2* tw, double2* out);

// MFCC tail: mel [B,T,M] dB values -> clamp(max - top_db) -> DCT [M,K] -> feats [B,T,K] + CMN partial sums.
struct MfccParams {
  const float* mel; const float* cta_max; const float* dct; float* feats; float* partial;
  int B, T, M, K, fpb, nblk, n_max;
  float top_db;        // < 0: no clamp
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

}  // namespace vpb
