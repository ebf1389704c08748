/* vpb200.h -- C ABI of the GPU-native speaker-embedding extraction path (H100, sm_90a).
 *
 * The reference (yeyupiaoling/VoiceprintRecognition-Pytorch, mvector 1.1.1) is pure Python and has NO FFI /
 * plugin boundary (SURVEY.md section 8b); the seam it offers is two Python callables:
 *     seam 1  AudioFeaturizer.forward(waveforms[, lens_ratio]) -> [B,T,F]   mvector/data_utils/featurizer.py:53-91
 *     seam 2  predictor(features) -> [B, embd_dim]                          mvector/predict.py:228,262
 * driven by MVectorPredictor.predict / predict_batch (mvector/predict.py:214-265).  This header is the C ABI a
 * maintainer binds (ctypes stub in INTEGRATION.md) to replace exactly those two callables:
 *     vp_fbank / vp_melspec   <-> seam 1 (KaldiFbank: featurizer.py:119-132 -> torchaudio kaldi.py:514-645;
 *                                          MelSpectrogram: featurizer.py:41-42,76; CMN + mask: featurizer.py:77-90)
 *     vp_embed                <-> seam 2 (nn.Sequential(build_model(...)).eval(), predict.py:54-63)
 *     vp_embed_wave           <-> seam 1 + seam 2 back to back (predict.py:256-262)
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

#define VP_ABI_VERSION 4

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

/* wave [B, Lpad] (zero padded to the batch max, predict.py:248-254) -> feats [B, T, F], T = vp_num_frames(Lpad).
 * keep_frames: device int32 [B] = round(len_i / Lmax * T) (featurizer.py:82-84) or NULL for no masking.
 * scratch: device floats, at least vp_frontend_scratch_floats(B, Lpad).
 * vp_fbank   = torchaudio.compliance.kaldi.fbank per utterance (featurizer.py:47-48,119-132): kind 0, post 0.
 * vp_melspec = torchaudio.transforms.MelSpectrogram, and Spectrogram with a pass-through bank (featurizer.py:41-44):
 *              kind 1, post 0.
 * vp_mfcc    = torchaudio.transforms.MFCC (featurizer.py:45-46): kind 1, post 1.  The top_db clamp uses the maximum
 *              over ALL B utterances of the call, as torchaudio does for a [B, n_mels, T] input. */
size_t vp_frontend_scratch_floats(const vp_handle* h, int32_t B, int32_t Lpad);
int vp_fbank(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats,
             float* scratch, void* stream);
int vp_melspec(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats,
               float* scratch, void* stream);
int vp_mfcc(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats,
            float* scratch, void* stream);

/* vp_mfcc in two stages, for callers that split ONE reference call over several processes (utterance sharding,
 * SURVEY.md 8e): the top_db clamp of torchaudio's MFCC uses the maximum over the WHOLE call, so a sharded call computes
 *   vp_mfcc_mel    : mel dB values of its shard into `scratch`, their maximum into max_out[0] (device float),
 *   (caller)       : all-reduce(MAX) of that one scalar over the ranks (ncclAllReduce / torch.distributed),
 *   vp_mfcc_finish : clamp to max_in[0] - top_db, DCT-II, CMN, mask -> feats.
 * `scratch` (vp_frontend_scratch_floats(B, Lpad) floats) must be left untouched between the two calls.
 * vp_mfcc == vp_mfcc_mel + vp_mfcc_finish with max_in = max_out. */
int vp_mfcc_mel(vp_handle* h, const float* wave, int32_t B, int32_t Lpad, float* scratch, float* max_out, void* stream);
int vp_mfcc_finish(vp_handle* h, int32_t B, int32_t Lpad, const int32_t* keep_frames, float* feats, float* scratch,
                   const float* max_in, void* stream);

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
enum { VP_ACT_NONE = 0, VP_ACT_RELU = 1, VP_ACT_HARDTANH20 = 2, VP_ACT_SIGMOID = 3, VP_ACT_TANH = 4, VP_ACT_SILU = 5 };
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
   * below 2^14, so the split is range-safe whatever the magnitude of the activations.  0 = none: the op then never runs
   * on the fp16 split (it stays on split-TF32, which has fp32's range). */
  int32_t amax_out, amax_in;
  /* Accumulation chunk of the tensor-core engines: 0 = the whole K extent goes into one accumulator; > 0 (a multiple of
   * 64) = every tc_kc K elements go into a fresh accumulator and the consumer warps fold the chunks with correctly
   * rounded fp32 adds.  The tensor core truncates on every accumulate (a bias that grows linearly with the chain
   * length); deep networks set a short chunk on their long-K layers.  A chunked op uses tc_bn <= 64 (second register set
   * for the running sum). */
  int32_t tc_kc;
  int32_t reserved0;
} vp_op;

/* Upload the packed fp32 weight arena (host pointer, copied to the device; replaces any previous arena). */
int vp_weights_load(vp_handle* h, const void* host_blob, size_t nbytes);

/* Validate + own a program for fixed (B, T).  Its workspace is the handle's shared arena, grown (after draining the
 * device) when workspace_bytes exceeds the current arena -- serving ragged lengths therefore costs max, not sum, of the
 * programs' workspaces, and destroying a program frees host memory only. */
int vp_program_create(vp_handle* h, const vp_op* ops, int32_t n_ops, size_t workspace_bytes, size_t input_floats,
                      size_t output_floats, vp_program** out);
void vp_program_destroy(vp_program* p);
/* feats [B,T,F] -> emb [B, embd_dim] */
int vp_embed(vp_program* p, const float* feats, float* emb, void* stream);
/* wave [B,Lpad] -> emb: front-end then program; feats_scratch holds B*T*F floats, fe_scratch as for vp_fbank */
int vp_embed_wave(vp_program* p, const float* wave, int32_t B, int32_t Lpad, const int32_t* keep_frames,
                  float* feats_scratch, float* fe_scratch, float* emb, void* stream);
/* Same as vp_embed but brackets every op with CUDA events on `stream`, synchronises, and writes the per-op device
 * time in milliseconds to the HOST array ms_per_op[n_ops] (bench.py's live roofline measurement). */
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
 * (infer_utils/speaker_diarization.py:254-257). */
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
/* number of kernel launches one vp_embed enqueues (bench.py's gpu_launches) */
int32_t vp_program_launches(const vp_program* p);
/* debugging / tests: copy a workspace region to a caller device buffer on the stream */
int vp_program_peek(vp_program* p, int64_t byte_offset, size_t nbytes, void* dst_device, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPB200_H_ */
