"""ctypes binding of libvpb200.so (include/vpb200.h).  Fails loudly when the CUDA library is missing: there is
no CPU / PyTorch fallback behind this module."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('VPB_LIB') or os.path.join(os.path.dirname(_HERE), 'libvpb200.so')   # VPB_LIB: dev builds

VP_OK, VP_ERR_INVALID, VP_ERR_CUDA, VP_ERR_NOMEM, VP_ERR_UNSUPPORTED = 0, 1, 2, 3, 4
OP_CONV, OP_CONV_C1, OP_COLSTATS, OP_ASP_POOL, OP_EW, OP_POOL2D = 1, 2, 3, 4, 5, 6
POOL_MAX, POOL_AVG = 0, 1
ACT_NONE, ACT_RELU, ACT_HARDTANH20, ACT_SIGMOID, ACT_TANH, ACT_SILU = 0, 1, 2, 3, 4, 5
PAD_ZERO, PAD_REFLECT = 0, 1
SRC2_NONE, SRC2_ADD, SRC2_CONCAT = 0, 1, 2
STATS_MEAN, STATS_MEAN_STD_CLAMP, STATS_MEAN_STD_UNBIASED, STATS_MEAN_STD_TSTP, STATS_SEG_CONTEXT = 0, 1, 2, 3, 4
STATS_MEAN_VAR_UNBIASED = 5
EW_GATE_RES, EW_AFF, EW_COPY, EW_PAD_COPY = 0, 1, 2, 3
BUF_NONE, BUF_INPUT, BUF_OUTPUT = -1, -2, -3
ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC, ENGINE_TC16 = 0, 1, 2, 3


class FrontendDesc(C.Structure):
    _fields_ = [('kind', C.c_int32), ('n_fft', C.c_int32), ('win_length', C.c_int32), ('hop', C.c_int32),
                ('n_mels', C.c_int32), ('remove_dc', C.c_int32), ('preemph', C.c_float), ('power', C.c_int32),
                ('use_log', C.c_int32), ('log_floor', C.c_float), ('post', C.c_int32), ('n_out', C.c_int32),
                ('db_mult', C.c_float), ('top_db', C.c_float)]


FRAME_DEFAULT, FRAME_KALDI_REFLECT, FRAME_STFT_CONSTANT, FRAME_STFT_REPLICATE, FRAME_STFT_CIRCULAR = 0, 1, 2, 3, 4
FRAME_STFT_NOCENTER = 5


class FrontendOptions(C.Structure):
    _fields_ = [('frame_mode', C.c_int32), ('pad', C.c_int32), ('spec_scale', C.c_double)]


class Op(C.Structure):
    _fields_ = ([('kind', C.c_int32), ('mode', C.c_int32), ('engine', C.c_int32), ('B', C.c_int32)]
                + [(n, C.c_int64) for n in ('src', 'src2', 'dst', 'res', 'gate', 'ubias',
                                            'w', 'bias', 'pre_s', 'pre_h', 'post_s', 'post_h', 'w_tc', 'sum')]
                + [(n, C.c_int32) for n in ('Tin', 'Fin', 'Cin', 'in_ld', 'in_coff',
                                            'src2_mode', 'src2_ld', 'src2_coff', 'Cin2',
                                            'Tout', 'Fout', 'Cout', 'out_ld', 'out_coff',
                                            'res_ld', 'res_coff',
                                            'KT', 'KF', 'sT', 'sF', 'dT', 'dF', 'padT', 'padF', 'pad_mode',
                                            'w_ld', 'pre_relu', 'act', 'act2', 'seg_len', 'n_seg')]
                + [('eps', C.c_float), ('tc_bn', C.c_int32), ('sum_ld', C.c_int32), ('sum_coff', C.c_int32),
                   ('w_tc16_q', C.c_int32), ('tc16_descale', C.c_float), ('amax_out', C.c_int32), ('amax_in', C.c_int32), ('tc_kc', C.c_int32), ('reserved0', C.c_int32)])


class VerifyResult(C.Structure):
    _fields_ = ([(n, C.c_int64) for n in ('n_target', 'n_impostor', 'x1', 'x2', 'target_x1', 'impostor_x1', 'target_x2',
                                          'impostor_x2')]
                + [('min_cost', C.c_double), ('argmin', C.c_int64), ('threshold', C.c_float), ('reserved0', C.c_int32)])


class VpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f'vpb200 error {code}: {msg}')
        self.code = code


_lib = None


def lib():
    """Load the shared library once.  Raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f'{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). '
                           'There is no CPU fallback for this path.')
    L = C.CDLL(LIB_PATH)
    vp, pp, i32, f32p, i32p, sz = C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t
    sig = {
        'vp_abi_version': (C.c_int, []),
        'vp_sizeof_op': (i32, []),
        'vp_sizeof_frontend_desc': (i32, []),
        'vp_sizeof_frontend_options': (i32, []),
        'vp_create': (C.c_int, [C.c_int, pp]),
        'vp_destroy': (None, [vp]),
        'vp_last_error': (C.c_char_p, [vp]),
        'vp_frontend_set': (C.c_int, [vp, C.POINTER(FrontendDesc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, i32, C.c_void_p]),
        'vp_frontend_set_options': (C.c_int, [vp, C.POINTER(FrontendOptions)]),
        'vp_feature_dim': (i32, [vp]),
        'vp_num_frames': (i32, [vp, i32]),
        'vp_frontend_scratch_floats': (sz, [vp, i32, i32]),
        'vp_fbank': (C.c_int, [vp, f32p, i32, i32, i32p, f32p, f32p, vp]),
        'vp_melspec': (C.c_int, [vp, f32p, i32, i32, i32p, f32p, f32p, vp]),
        'vp_mfcc': (C.c_int, [vp, f32p, i32, i32, i32p, f32p, f32p, vp]),
        'vp_mfcc_mel': (C.c_int, [vp, f32p, i32, i32, f32p, f32p, vp]),
        'vp_mfcc_finish': (C.c_int, [vp, i32, i32, i32p, f32p, f32p, f32p, vp]),
        'vp_weights_load': (C.c_int, [vp, C.c_void_p, sz]),
        'vp_program_create': (C.c_int, [vp, C.POINTER(Op), i32, sz, sz, sz, pp]),
        'vp_program_destroy': (None, [vp]),
        'vp_embed': (C.c_int, [vp, f32p, f32p, vp]),
        'vp_embed_wave': (C.c_int, [vp, f32p, i32, i32, i32p, f32p, f32p, f32p, vp]),
        'vp_program_launches': (i32, [vp]),
        'vp_embed_profiled': (C.c_int, [vp, f32p, f32p, vp, C.c_void_p]),
        'vp_program_op_info': (C.c_int, [vp, i32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        'vp_program_peek': (C.c_int, [vp, C.c_int64, sz, C.c_void_p, vp]),
        'vp_host_gather_pad': (C.c_int, [C.c_void_p, C.c_void_p, i32, i32, C.c_void_p, i32]),
        'vp_host_stage_h2d': (C.c_int, [C.c_void_p, C.c_void_p, i32, i32, C.c_void_p, C.c_void_p, i32, i32, vp]),
        'vp_host_gather_streaming': (C.c_int, [C.c_int]),
        'vp_workspace_bytes': (sz, [vp]),
        'vp_device_zero': (C.c_int, [C.c_void_p, sz, vp]),
        'vp_cosine_scores': (C.c_int, [vp, f32p, i32, f32p, i32, i32, f32p, vp]),
        'vp_spectral_scratch_bytes': (sz, [vp, i32]),
        'vp_spectral_laplacian': (C.c_int, [vp, f32p, i32, i32, i32, C.c_void_p, C.c_void_p, vp]),
        'vp_sym_tridiag': (C.c_int, [vp, C.c_void_p, i32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, vp]),
        'vp_sym_tridiag_apply_q': (C.c_int, [vp, C.c_void_p, C.c_void_p, i32, C.c_void_p, i32, vp]),
        'vp_spectral_launches': (i32, [i32]),
        'vp_verify_scratch_bytes': (sz, [vp, C.c_int64]),
        'vp_verify_metrics': (C.c_int, [vp, f32p, C.c_int64, i32p, i32p, C.c_int64, i32p, C.c_int64, C.c_double,
                                        C.c_double, C.c_double, C.c_void_p, f32p, C.c_void_p, C.c_void_p, vp]),
        'vp_resample': (C.c_int, [vp, f32p, C.c_int64, f32p, C.c_int64, i32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, vp]),
        'vp_gain_scratch_bytes': (sz, [vp, i32, C.c_int64]),
        'vp_gain_normalize': (C.c_int, [vp, f32p, C.c_int64, i32, C.c_void_p, C.c_double, C.c_double, C.c_void_p,
                                        C.c_void_p, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    if L.vp_abi_version() != 4:
        raise RuntimeError('libvpb200.so ABI version mismatch')
    if L.vp_sizeof_op() != C.sizeof(Op) or L.vp_sizeof_frontend_desc() != C.sizeof(FrontendDesc) \
            or L.vp_sizeof_frontend_options() != C.sizeof(FrontendOptions):
        raise RuntimeError('vp_op / vp_frontend_desc / vp_frontend_options layout mismatch between the ctypes binding '
                           'and libvpb200.so')
    _lib = L
    return L


EXPORTS = ['vp_abi_version', 'vp_sizeof_op', 'vp_sizeof_frontend_desc', 'vp_create', 'vp_destroy', 'vp_last_error',
           'vp_frontend_set', 'vp_sizeof_frontend_options', 'vp_frontend_set_options', 'vp_num_frames', 'vp_frontend_scratch_floats', 'vp_fbank', 'vp_melspec', 'vp_mfcc',
           'vp_feature_dim',
           'vp_weights_load', 'vp_program_create', 'vp_program_destroy', 'vp_embed', 'vp_embed_wave',
           'vp_program_launches', 'vp_program_peek', 'vp_embed_profiled', 'vp_program_op_info', 'vp_host_gather_pad',
           'vp_host_stage_h2d', 'vp_host_gather_streaming', 'vp_workspace_bytes', 'vp_mfcc_mel', 'vp_mfcc_finish', 'vp_cosine_scores', 'vp_device_zero',
           'vp_spectral_scratch_bytes', 'vp_spectral_laplacian', 'vp_sym_tridiag', 'vp_sym_tridiag_apply_q',
           'vp_spectral_launches', 'vp_verify_scratch_bytes', 'vp_verify_metrics',
           'vp_resample', 'vp_gain_scratch_bytes', 'vp_gain_normalize']
