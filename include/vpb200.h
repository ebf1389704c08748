/* vpb200.h -- C ABI of the GPU-native speaker-embedding extraction path (H100, sm_90a).
 *
 * The reference (yeyupiaoling/VoiceprintRecognition-Pytorch, mvector 1.1.1) is pure Python and has NO FFI /
 * plugin boundary (SURVEY.md section 8b); the seam it offers is two Python callables:
 *     seam 1  AudioFeaturizer.forward(waveforms[, lens_ratio]) -> [B,T,F]   mvector/data_utils/featurizer.py:53-91
 *     seam 2  predictor(features) -> [B, embd_dim]                          mvector/predict.py:228,262
 * driven by MVectorPredictor.predict / predict_batch (mvector/predict.py:214-265).  This header is the C ABI a
 * maintainer binds (ctypes stub in INTEGRATION.md) to replace exactly those two callables:
 *     vp_features             <-> seam 1 (KaldiFbank: featurizer.py:119-132 -> torchaudio kaldi.py:514-645;
 *                                          MelSpectrogram: featurizer.py:41-42,76; CMN + mask: featurizer.py:77-90)
 *     vp_embed                <-> seam 2 (nn.Sequential(build_model(...)).eval(), predict.py:54-63)
 *     vp_features + vp_embed  <-> seam 1 + seam 2 back to back (predict.py:256-262)
 *
 * Conventions: all tensor arguments are caller-owned DEVICE pointers to float32 (row-major, dense); every call
 * takes the CUDA stream to enqueue on (a cudaStream_t passed as void*, NULL = legacy default stream) and is
 * asynchronous; functions return 0 on success or a VP_ERR_* code, with vp_last_error() giving the message.
 * No hidden device allocation after vp_program_create.  One handle per device; thread-compatible: ONE thread and ONE
 * stream at a time per handle -- all programs of a handle share one workspace arena (sized to the largest of them), so
 * two programs of the same handle must never be in flight on different streams.  There is no CPU fallback anywhere
 * behind this ABI.
 */
#ifndef VPB200_H_
#define VPB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VP_ABI_VERSION 5

enum {
  VP_OK = 0,
  VP_ERR_INVALID = 1,      /* bad argument / inconsistent op */
  VP_ERR_CUDA = 2,         /* a CUDA runtime call failed (message has the cudaError string) */
  VP_ERR_NOMEM = 3,
  VP_ERR_UNSUPPORTED = 4   /* shape/option outside what the kernels implement; never silently emulated */
};

typedef struct vp_handle vp_handle;
typedef struct vp_program vp_program;

/* ------------------------------------------------------------------------------------------------------------
 * Front-end (seam 1).  kind 0 = Kaldi Fbank framing (per-frame DC removal, pre-emphasis, window, zero-pad to n_fft;
 * kaldi.py:154-217), kind 1 = torch.stft framing (frames of n_fft samples, functional.py:123-135).  Which samples a
 * frame takes (snip_edges or reflected edges; centred in one of four pad modes or not centred, after `pad` zeros) is
 * set by vp_frontend_set_options; vp_frontend_set selects the default framing of the kind.  Then |rFFT|^2 (power 2)
 * or |rFFT| (power 1), optionally scaled first (`normalized`), sparse triangular mel projection, optional
 * log(max(x, log_floor)), then (featurizer.py:77-90) time-mean subtraction over ALL T frames and zeroing of frames
 * >= keep_frames[b].
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct vp_frontend_desc {
  int32_t kind;         /* 0 kaldi-fbank framing, 1 centred-STFT framing */
  int32_t n_fft;        /* FFT size N = 2^a 3^b 5^c, multiple of 4, in [64, 2048] */
  int32_t win_length;   /* samples taken per frame (<= n_fft); window[] has this many taps */
  int32_t hop;          /* frame shift in samples */
  int32_t n_mels;       /* filter count, <= n_fft/2+1 (<= 1025): mel filters (<= 128 for MFCC) or Spectrogram bins */
  int32_t remove_dc;    /* kind 0: subtract the frame mean */
  float   preemph;      /* kind 0: pre-emphasis coefficient (0 = off) */
  int32_t power;        /* 2 = power spectrum, 1 = magnitude */
  int32_t use_log;      /* 0 none; 1 ln(max(x, log_floor)); 2 db_mult*log10(max(x, log_floor)); 3 ln(x + log_floor) */
  float   log_floor;
  int32_t post;         /* 0: the filter outputs are the features; 1: MFCC = DCT-II over the n_mels log values */
  int32_t n_out;        /* post 1: cepstral coefficients kept (<= n_mels); ignored otherwise */
  float   db_mult;      /* use_log 2 multiplier (10 for power, AmplitudeToDB) */
  float   top_db;       /* post 1: clamp the log values to (max over the whole call) - top_db first; < 0 = no clamp */
} vp_frontend_desc;

int vp_create(int device, vp_handle** out);
void vp_destroy(vp_handle* h);
const char* vp_last_error(const vp_handle* h);
int vp_abi_version(void);
int32_t vp_sizeof_op(void);             /* binding self-check: sizeof(vp_op) */
int32_t vp_sizeof_frontend_desc(void);  /* binding self-check: sizeof(vp_frontend_desc) */

/* window: win_length floats.  Mel bank in CSR-like form: filter m covers FFT bins
 * [mel_start[m], mel_start[m] + mel_count[m]) with weights mel_w[mel_off[m] ...]; dct: [n_mels, n_out] row-major
 * (torchaudio create_dct layout) when desc->post == 1, else NULL; all host pointers, copied. */
int vp_frontend_set(vp_handle* h, const vp_frontend_desc* desc, const float* window, const int32_t* mel_start,
                    const int32_t* mel_count, const int32_t* mel_off, const float* mel_w, int32_t n_w, const float* dct);

/* Framing and spectrum scale of the configured front-end.  vp_frontend_set resets them to the defaults
 * {VP_FRAME_DEFAULT, 0, 1.0}, which give kind 0 snip_edges framing and kind 1 centred reflect framing.  With L' = L + 2 pad:
 *   VP_FRAME_DEFAULT, kind 0   frames [t hop, t hop + win_length), T = 1 + (L - win_length) / hop       (snip_edges)
 *   VP_FRAME_KALDI_REFLECT     kind 0: T = (L + hop/2) / hop frames of the signal extended half-sample-symmetrically at
 *                              both ends, starting win_length/2 - hop/2 samples before x[0] (kaldi.py:44-83)
 *   VP_FRAME_DEFAULT, kind 1   T = 1 + L' / hop frames centred on t hop, the n_fft/2 samples beyond each end of the
 *                              zero-extended signal reflected (torch.stft center=True, pad_mode 'reflect')
 *   VP_FRAME_STFT_CONSTANT / _REPLICATE / _CIRCULAR   kind 1: the same with zeros, the edge sample, or wrap-around
 *   VP_FRAME_STFT_NOCENTER     kind 1: T = 1 + (L' - n_fft) / hop frames, no centring (center=False)
 * Each call fails with VP_ERR_INVALID before any launch when the waveform length breaks what torch requires:
 * kind 0: 2 <= win_length <= L; reflect: n_fft/2 < L'; circular: n_fft/2 <= L'; not centred: n_fft <= L'. */
enum { VP_FRAME_DEFAULT = 0, VP_FRAME_KALDI_REFLECT = 1, VP_FRAME_STFT_CONSTANT = 2, VP_FRAME_STFT_REPLICATE = 3,
       VP_FRAME_STFT_CIRCULAR = 4, VP_FRAME_STFT_NOCENTER = 5 };
typedef struct vp_frontend_options {
  int32_t frame_mode;   /* VP_FRAME_*: must fit the configured kind */
  int32_t pad;          /* kind 1: zeros added at both ends before framing (torchaudio `pad`); 0 for kind 0 */
  double  spec_scale;   /* kind 1: |X| multiplier before |.|^power (1/sqrt(sum w^2) or 1/sqrt(n_fft): `normalized`);
                           1.0 = none, the only value for kind 0 */
} vp_frontend_options;
int vp_frontend_set_options(vp_handle* h, const vp_frontend_options* opts);   /* after vp_frontend_set */
int32_t vp_sizeof_frontend_options(void);  /* binding self-check: sizeof(vp_frontend_options) */

/* feature dimension F the configured front-end emits (n_mels, or n_out for MFCC) */
int32_t vp_feature_dim(const vp_handle* h);
/* number of frames T the configured front-end yields for n_samples (kaldi.py:63-83 / torch.stft; see the framing above) */
int32_t vp_num_frames(const vp_handle* h, int32_t n_samples);

/* The configured front-end: wave [B, Lpad] (zero padded to the batch max, predict.py:248-254) -> feats [B, T, F],
 * T = vp_num_frames(Lpad).  keep_frames: device int32 [B] = round(len_i / Lmax * T) (featurizer.py:82-84) or NULL
 * for no masking.  scratch: device floats, at least vp_frontend_scratch_floats(B, Lpad).  What vp_frontend_set
 * configured decides which torchaudio call this is:
 *   kind 0, post 0: torchaudio.compliance.kaldi.fbank per utterance (featurizer.py:47-48,119-132);
 *   kind 1, post 0: torchaudio.transforms.MelSpectrogram, and Spectrogram with a pass-through bank
 *                   (featurizer.py:41-44);
 *   kind 1, post 1: torchaudio.transforms.MFCC (featurizer.py:45-46).  The top_db clamp uses the maximum over ALL B
 *                   utterances of the call, as torchaudio does for a [B, n_mels, T] input. */
size_t vp_frontend_scratch_floats(const vp_handle* h, int32_t B, int32_t Lpad);
int vp_features(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats,
                float* scratch, void* stream);

/* The configured front-end on a ragged batch, every row as if it were the whole call: the reference's eval /
 * feature-extraction mode (reader.py:82-107), which featurizes each file alone and zero-pads the features to the batch's
 * longest (collate_fn.py:5-24).
 *   wave  [B, ld] device floats, row b holding lens[b] samples (lens: device int32 [B], each in [0, ld])
 *   T     the frames of the longest row, vp_num_frames(max lens[b]); 1 <= T <= vp_num_frames(ld)
 *   feats [B, T, F]: row b's first T_b = vp_num_frames(lens[b]) frames are exactly what a one-row call on its lens[b]
 *         samples returns (framing at the row's own end, CMN over its own frames, MFCC's top_db clamp against its own
 *         maximum); frames T_b .. T-1 are +0.0.  Nothing is written past T.
 *   scratch: device floats, at least vp_frontend_scratch_floats(B, n) for n the longest row's lens (ld always does).
 * ld must pass the call's length check above; a row whose length breaks it gives unspecified features but reads no
 * sample outside its own first lens[b]. */
int vp_features_each(vp_handle* h, const float* wave, int32_t B, int32_t ld, const int32_t* lens, int32_t T, float* feats,
                     float* scratch, void* stream);

/* vp_features of the MFCC front-end in two stages, for callers that split ONE reference call over several processes
 * (utterance sharding, SURVEY.md 8e): the top_db clamp of torchaudio's MFCC uses the maximum over the WHOLE call, so a
 * sharded call computes
 *   vp_mfcc_mel    : mel dB values of its shard into `scratch`, their maximum into max_out[0] (device float),
 *   (caller)       : all-reduce(MAX) of that one scalar over the ranks (ncclAllReduce / torch.distributed),
 *   vp_mfcc_finish : clamp to max_in[0] - top_db, DCT-II, CMN, mask -> feats.
 * `scratch` (vp_frontend_scratch_floats(B, Lpad) floats) must be left untouched between the two calls.
 * vp_features == vp_mfcc_mel + vp_mfcc_finish with max_in = max_out. */
int vp_mfcc_mel(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, float* scratch, float* max_out, void* stream);
int vp_mfcc_finish(vp_handle* h, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats, float* scratch,
                   const float* max_in, void* stream);

/* Host only (no launch, no device access): how a call on B rows of Lpad samples runs frontend_kernel.  stage: 0 for a
 * vp_features call, 1 for the MFCC mel stage (it must match the configured front-end).  info[8] =
 *   [0] instantiation: the n_fft of the register-resident kernel (256, 512, 1024, 2048), 0 for the plan-driven one
 *   [1] G, threads per FFT group       [2] tpc, 16-frame tiles per CTA   [3] 1 when the CTA caches its features on chip
 *   [4] FFT passes                     [5] mel projection: 0 plain loop, 1 four interleaved chains
 *   [6] nblk, 16-frame tiles per row   [7] grid.x, CTAs per row
 * VP_ERR_INVALID when the call itself would be refused. */
int vp_frontend_plan_info(const vp_handle* h, int32_t B, int32_t Lpad, int32_t stage, int32_t* info);

/* ------------------------------------------------------------------------------------------------------------
 * Hugging Face wav2vec 2.0 / WavLM front-end (use_hf_model, featurizer.py:25-38,65-73).  The reference keeps only
 * `extract_features` of the model, which is the processor's normalisation followed by the convolutional feature encoder
 * and the feature projection's LayerNorm:
 *   x = do_normalize ? (w - mean(w)) / sqrt(var(w) + 1e-7) : w            numpy float32, per row (Wav2Vec2FeatureExtractor)
 *   h = conv_l(h), no padding, bias iff conv_bias, then
 *         norm 0 ("group"): layer 0 -> GroupNorm(one group per channel, over time, norm_eps) -> GELU; others -> GELU
 *         norm 1 ("layer"): every layer -> LayerNorm over channels (norm_eps) -> GELU
 *   f = LayerNorm(conv_dim[n - 1], proj_eps)(h)
 * then the CMN and keep mask of every front-end.  vp_frontend_set_hf makes this the configured front-end (replacing
 * any other, and vp_frontend_set replaces it): vp_features, vp_features_each, vp_frontend_scratch_floats,
 * vp_num_frames, vp_feature_dim and vp_frontend_plan_info then serve it; vp_mfcc_mel / vp_mfcc_finish and
 * vp_frontend_set_options refuse it.  The handle owns the encoder's weights (front-end state, not the backbone arena).
 *   frames: T_0 = n < k_0 ? 0 : (n - k_0) / s_0 + 1, T_l = T_{l-1} < k_l ? 0 : (T_{l-1} - k_l) / s_l + 1; a call needs
 *           T_{n-1} >= 1 (400 samples for the base geometry) and fails with VP_ERR_INVALID before any launch otherwise.
 *   layer 0 needs k_0 a multiple of s_0 (it runs as a k_0 / s_0-tap conv over rows of s_0 samples, s_0 <= 16); every
 *   layer's channels are multiples of 4 in [16, 1024].  The convolutions run on the split-TF32 tensor-core engine.
 *   Rows are independent: a row's features depend on its own samples and (padded call) the padded length only, never
 *   on the other rows or on the slicing below.  The call runs over slices of rows so that its scratch stays below
 *   VP_HF_SCRATCH_CAP floats (1 GiB) whatever B is (one row per slice when a single row needs more: about 80 s of
 *   16 kHz audio at 512 channels); vp_frontend_scratch_floats gives the exact need.
 * ---------------------------------------------------------------------------------------------------------- */
#define VP_HF_MAX_LAYERS 8
#define VP_HF_SCRATCH_CAP ((size_t)1 << 28)
enum { VP_HF_NORM_GROUP = 0, VP_HF_NORM_LAYER = 1 };
typedef struct vp_hf_desc {
  int32_t n_layers;                        /* conv layers, 1 .. VP_HF_MAX_LAYERS */
  int32_t conv_dim[VP_HF_MAX_LAYERS];      /* output channels of each layer */
  int32_t conv_kernel[VP_HF_MAX_LAYERS];
  int32_t conv_stride[VP_HF_MAX_LAYERS];
  int32_t conv_bias;                       /* 1: every conv has a bias */
  int32_t norm;                            /* VP_HF_NORM_* (feat_extract_norm) */
  int32_t do_normalize;                    /* 1: the processor's zero-mean unit-variance row normalisation */
  float   norm_eps;                        /* the conv layers' GroupNorm / LayerNorm eps (1e-5) */
  float   proj_eps;                        /* feature_projection.layer_norm eps (config.layer_norm_eps) */
} vp_hf_desc;
int32_t vp_sizeof_hf_desc(void);        /* binding self-check: sizeof(vp_hf_desc) */
/* Host pointers, copied: conv_w[l] is layer l's weight [conv_dim[l], C_in, conv_kernel[l]] (C_in = 1 for layer 0,
 * conv_dim[l-1] after), conv_b[l] its bias [conv_dim[l]] (NULL entries when !conv_bias); norm_w / norm_b[l] the affine
 * of layer l's norm (only [0] for norm 0); proj_w / proj_b the projection LayerNorm's [conv_dim[n - 1]]. */
int vp_frontend_set_hf(vp_handle* h, const vp_hf_desc* desc, const float* const* conv_w, const float* const* conv_b,
                       const float* const* norm_w, const float* const* norm_b, const float* proj_w, const float* proj_b);

/* ------------------------------------------------------------------------------------------------------------
 * Backbone (seam 2).  The host (Python mirror of the reference's mvector/models modules) lowers a model + a concrete (B, T) to a
 * straight-line program of fused ops over a workspace arena; weights live in one packed arena uploaded once.
 * Activations are channel-last: 1-D maps are [B, T, C], 2-D maps are [B, T, F, C] (T = time = conv2d W axis,
 * F = frequency = conv2d H axis of the reference's [B, C, F, T]).
 * ---------------------------------------------------------------------------------------------------------- */
enum {                       /* vp_op.kind */
  VP_OP_CONV = 1,            /* implicit-GEMM conv1d/conv2d/linear with fused prologue + epilogue */
  VP_OP_CONV_C1 = 2,         /* KTxKF (<= 7x7) strided conv2d with Cin = 1 on the feature map [B,T,F] -> [B,T',F',C] */
  VP_OP_COLSTATS = 3,        /* per-utterance column statistics over rows (mean / mean+std variants / segments) */
  VP_OP_ASP_POOL = 4,        /* softmax over T of logits, attentive mean + std (pooling.py:122-126); mode 1 = mean only (SAP, pooling.py:62-64) */
  VP_OP_EW = 5,              /* elementwise: gate*x + residual, AFF blend, copy */
  VP_OP_POOL2D = 6           /* KTxKF max / average pooling on a channel-last 2-D map (res2net.py:33-34,105); mode 0 = max
                                (implicit -inf padding), 1 = average with count_include_pad (zero padding, divide by KT*KF) */
};
enum { VP_ACT_NONE = 0, VP_ACT_RELU = 1, VP_ACT_HARDTANH20 = 2, VP_ACT_SIGMOID = 3, VP_ACT_TANH = 4, VP_ACT_SILU = 5,
       VP_ACT_GELU = 6 };          /* GELU: exact erf form 0.5 v (1 + erf(v / sqrt 2)), torch's approximate='none' */
enum { VP_PAD_ZERO = 0, VP_PAD_REFLECT = 1 };
enum { VP_SRC2_NONE = 0, VP_SRC2_ADD = 1, VP_SRC2_CONCAT = 2 };
enum {                       /* VP_OP_COLSTATS modes (op.mode) */
  VP_STATS_MEAN = 0,               /* out[b, c] = mean over rows                                  (ecapa_tdnn.py:79, resnet_se.py:58-60) */
  VP_STATS_MEAN_STD_CLAMP = 1,     /* [mean ; sqrt(clamp(sum((x-mean)^2)/R, eps))]                (pooling.py:91-94,108) */
  VP_STATS_MEAN_STD_UNBIASED = 2,  /* [mean ; sqrt(sum((x-mean)^2)/(R-1))]                        (campplus.py:27-33) */
  VP_STATS_MEAN_STD_TSTP = 3,      /* [mean ; sqrt(sum((x-mean)^2)/(R-1) + eps)]                  (pooling.py:140-148) */
  VP_STATS_SEG_CONTEXT = 4,        /* out[b, s, c] = mean over rows + mean over segment s (ceil)  (campplus.py:96-111) */
  VP_STATS_MEAN_VAR_UNBIASED = 5   /* [mean ; sum((x-mean)^2)/(R-1)]  (TemporalStatisticsPooling returns the VARIANCE, pooling.py:44-46) */
};
enum { VP_EW_GATE_RES = 0, VP_EW_AFF = 1, VP_EW_COPY = 2,
       VP_EW_PAD_COPY = 3 };  /* dst[r, 0:Cout] = (src[r, 0:Cin], zeros): any Cin / in_ld; Cout % 4 == 0 (odd feature dims) */
enum { VP_BUF_NONE = -1, VP_BUF_INPUT = -2, VP_BUF_OUTPUT = -3 };  /* special values for activation offsets */
enum { VP_ENGINE_AUTO = 0,   /* vp_op.engine: fastest eligible of the three below (TC16 > TC > FFMA) */
       VP_ENGINE_FFMA = 1,   /* exact fp32 FFMA kernels */
       VP_ENGINE_TC = 2,     /* wgmma, three-pass split TF32 */
       VP_ENGINE_TC16 = 3 }; /* wgmma, three-pass two-term FP16 split with dynamic power-of-two activation scaling */

typedef struct vp_op {
  int32_t kind;
  int32_t mode;            /* COLSTATS / EW sub-mode */
  int32_t engine;          /* VP_OP_CONV: VP_ENGINE_* */
  int32_t B;               /* utterances */
  /* activation operands: byte offsets into the program workspace, or VP_BUF_* */
  int64_t src, src2, dst, res, gate, ubias;
  /* weight-arena operands: byte offsets (or -1) */
  int64_t w, bias, pre_s, pre_h, post_s, post_h;
  /* optional tensor-core image of w (or -1): split-TF32 hi/lo planes, tiled [n_tile][k_block][hi|lo][tc_bn rows][32]
   * floats with the 16-byte chunks of every 128-byte row XOR-swizzled by (row & 7) -- the wgmma SWIZZLE_128B K-major
   * shared-memory image, so one bulk-async copy lands a pipeline stage (see conv_tc.cu, mvector/engine.py::pack_tc) */
  int64_t w_tc;
  /* optional accumulate-into view (or VP_BUF_NONE): after the epilogue, sum[m, sum_coff + n] += y[m, n].  Lets a Res2
   * chain hand "x_{j+1} + y_j" to the next conv as ONE source (in place over x_{j+1}) instead of gathering two. */
  int64_t sum;
  /* source geometry: rows = B*Tin*Fin, each row in_ld floats, channels [in_coff, in_coff+Cin) */
  int32_t Tin, Fin, Cin, in_ld, in_coff;
  int32_t src2_mode, src2_ld, src2_coff, Cin2;   /* ADD: same Cin; CONCAT: channels Cin..Cin+Cin2 come from src2 */
  /* destination geometry: rows = B*Tout*Fout, row out_ld floats, channels [out_coff, out_coff+Cout) */
  int32_t Tout, Fout, Cout, out_ld, out_coff;
  int32_t res_ld, res_coff;
  /* taps (time, freq), strides, dilations, paddings */
  int32_t KT, KF, sT, sF, dT, dF, padT, padF, pad_mode;
  int32_t w_ld;            /* floats per weight row; weight element (n, (kt*KF+kf)*CinTot + ci) */
  int32_t pre_relu;        /* prologue: a = relu(a*pre_s[ci] + pre_h[ci]) when pre_s >= 0 (campplus.py:141-149) */
  int32_t act, act2;       /* y = act2(act(acc + bias + ubias) * post_s + post_h) * gate + res)  -- see DESIGN.md */
  int32_t seg_len, n_seg;  /* gate / ubias / SEG_CONTEXT rows per utterance: row (b*n_seg + min(t/seg_len, n_seg-1)) */
  float   eps;
  int32_t tc_bn;           /* N tile of w_tc: 128 (64 if tc_kc > 0) when Cout is at least that, else Cout rounded up to 16 */
  int32_t sum_ld, sum_coff;
  /* fp16 two-term image of w for the f16 variant of the tensor-core engine (VP_ENGINE_TC16; VPB_TC_F16=0 disables it
   * at run time).  w_tc16_q = (byte offset in the weight arena >> 4) + 1, 0 = none; layout
   * [n_tile][k_block of 64][hi|lo][tc_bn rows][64 halves], 16-byte chunks XOR-swizzled by (row & 7); the image holds
   * w * 2^k, tc16_descale = 2^-k is applied to the accumulator. */
  int32_t w_tc16_q;
  float   tc16_descale;
  /* Dynamic activation range for the fp16 split: "amax slots" are uint32 words (float bits, zeroed at the start of
   * every vp_embed) behind the program workspace.  An op with amax_out = s + 1 atomically maxes |y| over everything it
   * writes into slot s (max is exact and order independent: results stay deterministic); a CONV with amax_in = s + 1 may
   * run on the fp16 split and then scales its gathered activations by the power of two that puts slot s's maximum just
   * below 2^14, so the split keeps its accuracy for a slot maximum anywhere from 2^-113 up to the largest finite float.
   * (Below 2^-113 the scale would leave fp32's normal range; such a tensor's products lie among fp32's subnormals,
   * where the fp32 reference itself has lost bits.)  0 = none: the op then never runs on the fp16 split (it stays on
   * split-TF32, which has fp32's range). */
  int32_t amax_out, amax_in;
  /* Accumulation chunk of the tensor-core engines: 0 = the whole K extent goes into one accumulator; > 0 (a multiple of
   * 64) = every tc_kc K elements go into a fresh accumulator and the consumer warps fold the chunks with correctly
   * rounded fp32 adds.  The tensor core truncates on every accumulate (a bias that grows linearly with the chain
   * length); deep networks set a short chunk on their long-K layers.  A chunked op uses tc_bn <= 64 (second register set
   * for the running sum). */
  int32_t tc_kc;
  int32_t reserved0;
} vp_op;

/* Upload the packed fp32 weight arena (host pointer, copied to the device; replaces any previous arena).  Programs
 * created before the call -- whether it succeeds or not -- are validated against the old arena: vp_embed and
 * vp_embed_profiled refuse them with VP_ERR_INVALID before launching anything. */
int vp_weights_load(vp_handle* h, const void* host_blob, size_t nbytes);

/* Validate + own a program for fixed (B, T).  Its workspace is the handle's shared arena, grown (after draining the
 * device) when workspace_bytes exceeds the current arena -- serving ragged lengths therefore costs max, not sum, of the
 * programs' workspaces, and destroying a program frees host memory only. */
int vp_program_create(vp_handle* h, const vp_op* ops, int32_t n_ops, size_t workspace_bytes, size_t input_floats,
                      size_t output_floats, vp_program** out);
void vp_program_destroy(vp_program* p);
/* feats [B,T,F] -> emb [B, embd_dim] */
int vp_embed(vp_program* p, const float* feats, float* emb, void* stream);
/* Same as vp_embed but brackets every op with CUDA events on `stream`, synchronises, and writes the per-op device
 * time in milliseconds to the HOST array ms_per_op[n_ops] (bench.py's live roofline measurement).  Ops that run as one
 * launch -- a Res2Net chain of split-TF32 convs fused by vp_program_create -- book the launch's time on the chain's
 * first op and about 0 on the others. */
int vp_embed_profiled(vp_program* p, const float* feats, float* emb, void* stream, float* ms_per_op);
/* op i of the program: kind, GEMM view (M rows, N = Cout, K = taps*Cin; K = 0 for non-conv ops), resolved engine */
int vp_program_op_info(const vp_program* p, int32_t i, int32_t* kind, int64_t* M, int64_t* N, int64_t* K, int32_t* engine);
/* Host utility (no CUDA): gather n waveforms (host pointers srcs[i], lens[i] samples) into the zero-padded row-major
 * staging matrix dst[n, lmax] with n_threads worker threads -- the pad-to-longest loop of predict.py:248-254. */
int vp_host_gather_pad(const float* const* srcs, const int32_t* lens, int32_t n, int32_t lmax, float* dst,
                       int32_t n_threads);
/* cudaMemsetAsync(device_ptr, 0, nbytes) on `stream`: zero padding of feature batches by hosts that must not bring
 * their own kernels (collate_fn.py:12-19 pads FEATURES, not waveforms). */
int vp_device_zero(void* device_ptr, size_t nbytes, void* stream);

/* Cosine score matrix scores[i, j] = <a_i, b_j> / (|a_i| |b_j|), a [n, D], b [m, D], scores [n, m] (device, row-major):
 * the scoring step of the callers around the embedding path -- retrieval against the enrolled speaker means
 * (predict.py:169-183), evaluate's trial-vs-enrol scores (trainer.py:454-461) and the diarization similarity matrix
 * (infer_utils/speaker_diarization.py:254-257).  A zero-norm row scores +0 against every row, itself included, as
 * sklearn's cosine_similarity normalises a zero row to zero; a row holding a NaN gives NaN in its own row or column
 * only.  Any n, m, D >= 1; a score depends only on its two rows, not on n, m or its place in the matrix. */
int vp_cosine_scores(vp_handle* h, const float* a, int32_t n, const float* b, int32_t m, int32_t D, float* scores, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Spectral stage of the diarization clustering: SpectralCluster.__call__ (infer_utils/speaker_diarization.py:235-250)
 * up to its eigenvectors, in fp64 after the affinity.  The tridiagonal eigenproblem in between (2n numbers down, [n, k]
 * up) is the caller's: mvector/engine.py::spectral_embedding solves it with LAPACK stebz/stein.
 * ---------------------------------------------------------------------------------------------------------- */
/* device scratch bytes that vp_spectral_laplacian and vp_sym_tridiag need for an n-point problem (n^2 floats at most) */
size_t vp_spectral_scratch_bytes(const vp_handle* h, int32_t n);
/* emb [n, D] float32 -> L [n, n] float64 (row-major, both triangles), the unnormalised Laplacian of the pruned affinity:
 *   S0 = cosine(emb, emb)                       (get_sim_mat, :253-257; the vp_cosine_scores kernel)
 *   P  = S0 with the n_drop smallest entries of every row set to 0   (p_pruning, :260-274); ties at the cut go by column
 *        index, lower indices first (numpy's stable argsort; the reference's default quicksort leaves that order open)
 *   S  = 0.5 (P + P') in fp64, zero diagonal; d_i = sum_j |S_ij|; L = diag(d) - S   (:246, get_laplacian :277-283)
 * n_drop = len(range(n)[:int((1 - pval) * n)]) as Python evaluates p_pruning's expression, in [0, n).  n <= 58 000. */
int vp_spectral_laplacian(vp_handle* h, const float* emb, int32_t n, int32_t D, int32_t n_drop, double* L, void* scratch,
                          void* stream);
/* In-place Householder reduction of a symmetric A [n, n] (float64, full storage) to T = Q' A Q = tridiag(d, e), LAPACK
 * dsytd2 with UPLO = 'L': H_k = I - tau[k] v v', v = (0.., 1, A[k+2:, k]), beta = -sign(alpha) ||x||.  On return the
 * diagonal and first subdiagonal of A hold d and e, the strictly lower part below it the reflectors; the upper triangle
 * is scratch.  d [n], e [n-1], tau [n-1] (tau[n-2] = 0) are device float64.  Replaces the dense scipy.linalg.eigh of
 * get_spec_embs (:285-295) up to the tridiagonal eigenproblem. */
int vp_sym_tridiag(vp_handle* h, double* A, int32_t n, double* d, double* e, double* tau, void* scratch, void* stream);
/* Z [n, k] (float64, row-major, device) <- Q Z with the reflectors vp_sym_tridiag left in A and tau: eigenvectors of T
 * become eigenvectors of the original matrix.  1 <= k <= min(n, 16) (get_spec_embs keeps <= max_num_spks = 15 columns). */
int vp_sym_tridiag_apply_q(vp_handle* h, const double* A, const double* tau, int32_t n, double* Z, int32_t k,
                           void* stream);
/* kernel launches of one vp_spectral_laplacian + vp_sym_tridiag + vp_sym_tridiag_apply_q at size n */
int32_t vp_spectral_launches(int32_t n);

/* ------------------------------------------------------------------------------------------------------------
 * Verification metrics of MVectorTrainer.evaluate (trainer.py:462-468, metric/metrics.py:5-39) on the device: EER,
 * minDCF and the EER threshold of n scores, without copying the scores or building a label matrix on the host.
 * With order = argsort(scores, kind='stable') and T_i / I_i the inclusive counts of targets (label 1) / impostors
 * (label 0) among the first i+1 sorted scores, T = T_{n-1}, I = I_{n-1}:
 *   fnr[i] = T_i / T,  fpr[i] = 1 - I_i / I,  gap[i] = fnr[i] - fpr[i],
 *   cost[i] = ((c_miss * fnr[i]) * p_target) + ((c_fa * fpr[i]) * (1 - p_target))
 * in float64 with every operation rounded on its own (no FMA) -- the values numpy's compute_fnr_fpr / compute_dcf form.
 * Equal scores keep their index order (stable sort; the reference's default quicksort leaves that order open); -0 sorts
 * as +0 and every NaN after +inf, as numpy sorts them.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct vp_verify_result {
  int64_t n_target;        /* T: scores with label 1 */
  int64_t n_impostor;      /* I: scores with label 0 (any other flat label counts as neither) */
  int64_t x1;              /* first sorted index with gap >= 0, -1 if none (compute_eer's x1) */
  int64_t x2;              /* last sorted index with gap < 0, -1 if none (compute_eer's x2) */
  int64_t target_x1;       /* T_{x1} (0 if x1 = -1) */
  int64_t impostor_x1;     /* I_{x1} */
  int64_t target_x2;       /* T_{x2} (0 if x2 = -1) */
  int64_t impostor_x2;     /* I_{x2} */
  double  min_cost;        /* min over i of cost[i] (compute_dcf's c_det before the division by c_def) */
  int64_t argmin;          /* first index attaining min_cost, -1 if n = 0 */
  float   threshold;       /* sorted score at x1 (compute_eer's threshold; NaN if x1 = -1) */
  int32_t reserved0;
} vp_verify_result;
/* device scratch bytes vp_verify_metrics needs for n scores: about 10.3 bytes per score */
size_t vp_verify_scratch_bytes(const vp_handle* h, int64_t n);
/* scores [n] float32 (device, caller-owned; not modified), 0 <= n <= 2^31, and EITHER labels [n] int32 (flat form, as
 * compute_fnr_fpr takes them: 1 target, 0 impostor) with trial_labels = enroll_labels = NULL, OR labels = NULL and
 * trial_labels [n_trials] / enroll_labels [n_enroll] int32 with n = n_trials * n_enroll: score i is trial i / n_enroll
 * against enrolment i % n_enroll and a target iff their labels are equal (evaluate's trial-major matrix).
 * sorted_scores [n] float32 / sorted_labels [n] uint8 (1 target, 0 impostor, 2 neither) receive the sorted sequence
 * when not NULL.  result: DEVICE pointer to one vp_verify_result, valid once the stream reaches the end of the call.
 * All launches are asynchronous; no floating-point atomics: two calls give bit-identical results. */
int vp_verify_metrics(vp_handle* h, const float* scores, int64_t n, const int32_t* labels, const int32_t* trial_labels,
                      int64_t n_trials, const int32_t* enroll_labels, int64_t n_enroll, double p_target, double c_miss,
                      double c_fa, void* scratch, float* sorted_scores, uint8_t* sorted_labels, vp_verify_result* result,
                      void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Input conditioning of _load_audio (predict.py:185-212) on the device: resample to the model's rate, then dB-normalise.
 * ---------------------------------------------------------------------------------------------------------- */
/* Polyphase resampler: row b of out [B, out_ld] <- scipy.signal.resample_poly(in[b, :n_in[b]].astype(float64),
 * up[b], down[b]) (window ('kaiser', 5.0), padtype 'constant') rounded to float32; columns >= n_out[b] are written as 0.
 * n_out[b] must be ceil(n_in[b] * up[b] / down[b]) (in int64) and <= out_ld; up[b] == down[b] copies the row.
 * With max_rate = max(up, down), half_len = 10 max_rate, h = firwin(2 half_len + 1, 1 / max_rate, ('kaiser', 5.0)) * up,
 * n_pre_pad = down - half_len % down, hpad = (n_pre_pad zeros, h), Lh = len(hpad), nt = ceil(Lh / up) and
 * n_pre_remove = (half_len + n_pre_pad) / down, taps[tap_off[b] + p * nt + m] = hpad[p + m * up] (0 past Lh) for every
 * phase 0 <= p < up (float64, device; the host designs it once per (up, down)).  Output j is upfirdn output
 * i = j + n_pre_remove: acc = 0.0, then for k = max(0, ceil((i down - (Lh - 1)) / up)) .. min(n_in - 1, floor(i down / up))
 * in increasing order acc = __dadd_rn(acc, __dmul_rn((double)in[k], hpad[i down - k up])), one rounding to float32 at the
 * end: scipy's operation order, so the result is bit-identical.  n_in, n_out, tap_off int64 [B], up, down int32 [B],
 * all device.  in and out must not overlap.  Asynchronous on stream. */
int vp_resample(vp_handle* h, const float* in, int64_t in_ld, float* out, int64_t out_ld, int32_t B, const int64_t* n_in,
                const int64_t* n_out, const int32_t* up, const int32_t* down, const int64_t* tap_off, const double* taps,
                void* stream);
/* device scratch bytes vp_gain_normalize needs for B rows of leading dimension ld */
size_t vp_gain_scratch_bytes(const vp_handle* h, int32_t B, int64_t ld);
/* In place on wave [B, ld] (device float32), the twin of AudioSegment.normalize(target_db, max_gain_db) on
 * wave[b, :lens[b]] (lens int64 [B], device): mean = sum x^2 / n in float64 (per-tile sums of the exact squares combined
 * in tile order), gain = target_db - 10 log10(mean), factor = 10^(gain / 20) in float64 and x <- (float)(x * factor),
 * the float64 product numpy forms for a float32 array times a float64 scalar.  log10 / pow are CUDA's (<= 2 ulp from
 * glibc's), so a factor may differ from the host's in the last float64 bits; an output sample then differs by at most
 * one float32 ulp, and only when x * factor lies next to a float32 rounding boundary.  flags[b] (int32, device) <- 1
 * when gain > max_gain_db (a silent row: gain +inf), the row then left unscaled; else 0.  NaN samples give a NaN row,
 * as on the host.  Columns >= lens[b] are not touched.  Asynchronous on stream; no atomics. */
int vp_gain_normalize(vp_handle* h, float* wave, int64_t ld, int32_t B, const int64_t* lens, double target_db,
                      double max_gain_db, int32_t* flags, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Front of speaker_diarization (predict.py:365-379) on one device copy of the conditioned recording: the energy VAD's
 * frame energies (mvector/audio.py, AudioSegment.vad) and the chunk rows (SpeakerDiarization._chunk).
 * ---------------------------------------------------------------------------------------------------------- */
/* out[f] (float64, device) <- (wave[:nf*hop].astype(float64).reshape(nf, hop) ** 2).mean(axis=1)[f] for f < nf = n / hop,
 * bit-identical to numpy: each row is summed in numpy's pairwise order (below 8 elements sequentially from 0.0; up to 128
 * with eight strided accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail in order; above 128
 * split at n2 = n/2 - (n/2) % 8 and the halves added) with __dadd_rn, then one __ddiv_rn by hop.  wave: n float32
 * samples (device).  1 <= hop < 2^31; n < hop writes nothing.  NaN / inf propagate as in numpy.  Asynchronous on stream;
 * no atomics. */
int vp_frame_energy(vp_handle* h, const float* wave, int64_t n, int64_t hop, double* out, void* stream);
/* dst[i, j] (float32 [n, ld], device) <- j < valid[i] ? src[offset[i] + j] : 0 for j < ld: window i of the device row
 * src, zero filled past valid[i].  offset int64 [n], valid int32 [n], both device; src[offset[i] .. offset[i] +
 * min(valid[i], ld)) must lie inside src (offsets past 2^31 elements are fine).  src and dst must not overlap.
 * Asynchronous on stream. */
int vp_gather_windows(vp_handle* h, const float* src, const int64_t* offset, const int32_t* valid, int64_t n, int64_t ld,
                      float* dst, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * FLAC decoding (RFC 9639) of B native streams on the device, 4-24 bits per sample, 1-8 channels, every frame and
 * subframe coding the RFC defines for those depths.  CRC-8 is checked on every frame header and CRC-16 on every frame;
 * the STREAMINFO MD5 of the audio is not checked.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct vp_flac_info {  /* a stream's STREAMINFO (mvector/flac.py parses it on the host) */
  int64_t total_samples;       /* samples per channel, >= 1 (0 = unknown is not accepted) */
  int32_t sample_rate;
  int32_t channels;            /* 1..8 */
  int32_t bps;                 /* bits per sample, 4..24 */
  int32_t min_blocksize;       /* >= 16 */
  int32_t max_blocksize;       /* min_blocksize..65535 */
  int32_t min_framesize;       /* bytes, 0 = unknown */
  int32_t max_framesize;       /* bytes, 0 = unknown */
  int32_t reserved0;
} vp_flac_info;
int32_t vp_sizeof_flac_info(void);   /* binding self-check: sizeof(vp_flac_info) */
/* Device scratch bytes of one vp_flac_decode: about 5 bytes per input byte plus 8 per frame slot.  max_frames: the frame
 * slots of the batch, at least the sum over its streams of ceil(total_samples / min_blocksize). */
size_t vp_flac_scratch_bytes(const vp_handle* h, int32_t B, int64_t nbytes, int64_t max_frames);
/* data: the nbytes concatenated bytes of the B streams (device); the scan pass and the scratch cover exactly nbytes, so a
 * batch whose stream_off is not ordered inside [0, nbytes] has every stream refused (status 1) before any stream byte is
 * read.  stream_off int64 [B + 1]: stream b is data[stream_off[b] .. stream_off[b + 1]); frame_off int64 [B]: absolute offset of its first frame (the byte after its
 * last metadata block); info [B]: its STREAMINFO.  All device.
 * out [B, ld] float32 (device): row b <- the stream decoded, the channels of each sample mixed exactly as
 * mvector.audio.pcm_to_mono mixes the same integers (x / 2^(bps-1) in float32, then numpy's float32 mean over the
 * channels: left to right below 8 channels, ((c0+c1)+(c2+c3))+((c4+c5)+(c6+c7)) for 8, one division by the count; the
 * stereo decorrelations first), zero filled from total_samples to ld.
 * status int32 [B] (device) <- 0, or a non-zero OR of reasons: 1 STREAMINFO out of range (or total_samples > ld, or the
 * frame table would pass max_frames, or stream_off out of order or past nbytes), 2 no frame proven at frame_off, 4 frames that do not tile [0, total_samples)
 * exactly, 8 a frame header contradicting STREAMINFO, 16 a subframe with a reserved code, an out-of-range value or a
 * decode that does not end at the frame's CRC-16.  A refused row's samples are unspecified; the other rows are exact.
 * Every read of a stream stays inside its own byte range.  Asynchronous on stream. */
int vp_flac_decode(vp_handle* h, const uint8_t* data, const int64_t* stream_off, const int64_t* frame_off,
                   const vp_flac_info* info, int32_t B, float* out, int64_t ld, int32_t* status, void* scratch,
                   int64_t nbytes, int64_t max_frames, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Uncompressed PCM containers (WAV, WAVE_FORMAT_EXTENSIBLE, RF64 / BW64, AIFF / AIFF-C): B rows of raw interleaved
 * samples converted on the device.  mvector/pcm.py parses the headers on the host; the device reads only sample bytes.
 * Row b is float32 mono at the file's native rate, bit-identical to mvector.pcm.to_mono:
 *   integers of container width N bits (U8 is WAV's unsigned 8-bit, S8 AIFF's signed): x / 2^(N-1) in float32, exactly
 *     mvector.audio.pcm_to_mono (32-bit: float32(x) rounded to nearest first);
 *   F32: the stored value, no scaling or clipping; F64: rounded to nearest float32;
 *   ULAW / ALAW: the ITU-T G.711 expansion to a 16-bit integer (extremes +-32124 / +-32256), then / 2^15;
 *   channels 1..8: numpy's float32 mean -- left to right below 8 channels, ((c0+c1)+(c2+c3))+((c4+c5)+(c6+c7)) for 8,
 *     then one division by the count (the order vp_flac_decode uses).
 * ---------------------------------------------------------------------------------------------------------- */
enum {
  VP_PCM_U8 = 1, VP_PCM_S8 = 2, VP_PCM_S16LE = 3, VP_PCM_S16BE = 4, VP_PCM_S24LE = 5, VP_PCM_S24BE = 6,
  VP_PCM_S32LE = 7, VP_PCM_S32BE = 8, VP_PCM_F32LE = 9, VP_PCM_F32BE = 10, VP_PCM_F64LE = 11, VP_PCM_F64BE = 12,
  VP_PCM_ULAW = 13, VP_PCM_ALAW = 14
};
typedef struct vp_pcm_info {  /* where a row's samples are and how they are stored */
  int64_t byte_off;            /* offset of the first sample byte in data */
  int64_t frames;              /* samples per channel, 0..ld */
  int32_t channels;            /* 1..8, interleaved */
  int32_t format;              /* VP_PCM_* */
  int32_t reserved0;
  int32_t reserved1;
} vp_pcm_info;
int32_t vp_sizeof_pcm_info(void);    /* binding self-check: sizeof(vp_pcm_info) */
/* data: nbytes bytes (device, any alignment; may be null when nbytes is 0); info [B] (device); B in [0, 65535].
 * out [B, ld] float32 (device; may be null when ld is 0): row b at out + b * ld <- its frames converted as above, zero filled from frames to ld.
 * status int32 [B] (device) <- 0, or an OR of reasons checked before any of the row's bytes is read: 1 unknown format,
 * 2 channels outside 1..8, 4 frames outside [0, ld], 8 sample bytes [byte_off, byte_off + frames * channels * width)
 * not inside [0, nbytes).  A refused row is written as zeros; the other rows are exact.  Every read of a row stays
 * inside its own sample bytes.  Asynchronous on stream. */
int vp_pcm_decode(vp_handle* h, const uint8_t* data, int64_t nbytes, const vp_pcm_info* info, int32_t B, float* out,
                  int64_t ld, int32_t* status, void* stream);

/* Staging half of predict_batch (predict.py:244-255) as ONE native call: worker threads gather slices of slice_rows
 * utterances into the zero-padded PINNED matrix staging[n, lmax]; the calling thread -- one of the n_threads gatherers --
 * issues cudaMemcpyAsync(staging slice -> device_dst slice) on copy_stream, in slice order, as soon as a slice is
 * complete, so the H2D transfer of slice k overlaps the gather of slice k+1 (also with n_threads == 1).  Returns when the
 * last copy has been ENQUEUED.  device_dst == NULL: gather only (== vp_host_gather_pad). */
int vp_host_stage_h2d(const float* const* srcs, const int32_t* lens, int32_t n, int32_t lmax, float* staging,
                      float* device_dst, int32_t slice_rows, int32_t n_threads, void* copy_stream);
/* Process-wide switch of the staging gather: on != 0 -> rows are written with non-temporal (streaming) stores, which skip
 * the read-for-ownership of the pinned destination lines (the copy engine, not a CPU, reads them next): less DRAM traffic
 * when several ranks of one host stage at the same time.  Returns 1 when streaming stores are in effect (x86-64 with AVX2
 * or AVX-512), 0 otherwise (plain memcpy).  on < 0: query only. */
int vp_host_gather_streaming(int on);
/* bytes of the handle's shared workspace arena right now */
size_t vp_workspace_bytes(const vp_handle* h);
/* number of kernel launches one vp_embed enqueues (bench.py's gpu_launches): a fused Res2Net chain counts once */
int32_t vp_program_launches(const vp_program* p);
/* debugging / tests: copy a region of the program's workspace, or of the amax slots behind it (uint32 slot q at byte
 * offset round_up(workspace_bytes, 256) + 4 (q - 1)), to a caller device buffer on the stream */
int vp_program_peek(vp_program* p, int64_t byte_offset, size_t nbytes, void* dst_device, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPB200_H_ */
