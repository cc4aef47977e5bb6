"""ctypes binding of libpgt_b200.so (the C ABI declared in include/pgt_b200.h).

There is NO fallback: if the library is missing (and cannot be built) or a call fails, a
RuntimeError is raised.  PyTorch is used only for device memory and the current stream.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'lib', 'libpgt_b200.so')

BF16, F32 = 0, 1
ACT_NONE, ACT_GELU, ACT_SILU, ACT_LRELU02, ACT_RELU, ACT_SIGMOID = 0, 1, 2, 3, 4, 5
EPI_PLAIN, EPI_SFT = 0, 1
OUT_NHWC, OUT_NCHW = 0, 1


class Epilogue(Structure):
    _fields_ = [('bias', c_void_p), ('act', c_int32), ('mode', c_int32), ('residual', c_void_p),
                ('ldr', c_int32), ('res_dtype', c_int32), ('aux', c_void_p), ('ldaux', c_int32),
                ('sft_w', c_float), ('out', c_void_p), ('ldo', c_int32), ('out_dtype', c_int32),
                ('out_layout', c_int32), ('flags', c_int32), ('gn_stats', c_void_p), ('sft_wf', c_void_p)]


# name -> (restype, argtypes); mirrors include/pgt_b200.h one to one
SIGNATURES = {
    'pgt_strerror': (c_char_p, [c_int]),
    'pgt_last_cuda_error': (c_char_p, []),
    'pgt_version': (c_int, []),
    'pgt_launch_count': (c_int64, []),
    'pgt_reset_launch_count': (None, []),
    'pgt_tmap_cache_stats': (None, [c_void_p, c_void_p]),
    'pgt_profile_begin': (c_int, []),
    'pgt_profile_end': (c_int, [c_void_p, c_void_p, c_void_p]),
    'pgt_profile_end_csv': (c_int, [c_char_p, c_void_p, c_void_p, c_void_p]),
    'pgt_linear_bf16': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, POINTER(Epilogue), c_void_p]),
    'pgt_conv_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int,
                              c_int, POINTER(Epilogue), c_void_p]),
    'pgt_conv_out_gn': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                c_void_p, c_void_p]),
    'pgt_conv_out_gn_act': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                    c_void_p, c_void_p, c_int, c_void_p]),
    'pgt_groupnorm_ab': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int,
                                 c_void_p, c_void_p, c_void_p]),
    'pgt_conv_up2x_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                   POINTER(Epilogue), c_void_p]),
    'pgt_conv_rgb_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_groupnorm_ws_floats': (c_int64, [c_int, c_int, c_int]),
    'pgt_conv_tiles_per_frame': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    'pgt_conv_tiles_exact': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    'pgt_groupnorm_apply_stats': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int,
                                          c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_groupnorm_silu': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int,
                                   c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_layernorm': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int,
                              c_void_p, c_int, c_void_p, c_int, c_void_p]),
    'pgt_ln_linear_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int,
                                   c_void_p, c_void_p, c_int, c_void_p]),
    'pgt_swin_mlp_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_window_attention': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                     c_int, c_void_p]),
    'pgt_window_attention_tc': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                        c_int, c_void_p]),
    'pgt_window3d_attention': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    'pgt_mha_fwd': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                            c_int, c_void_p]),
    'pgt_argmax_gather': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_void_p]),
    'pgt_l2_argmin': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'pgt_codebook_pack': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'pgt_l2_argmin_ws_ints': (c_int64, [c_int]),
    'pgt_l2_argmin_tc': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    'pgt_l2_argmin_split_ws_ints': (c_int64, [c_int, c_int]),
    'pgt_l2_argmin_tc_split': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    'pgt_soft_codes': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_void_p, c_int, c_void_p]),
    'pgt_sample_codes': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'pgt_rq_residual': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    'pgt_rq_embed': (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_int, c_void_p, c_int,
                             c_int, c_void_p]),
    'pgt_vq_stats_ws_doubles': (c_int64, [c_int, c_int]),
    'pgt_vq_stats': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'pgt_adain': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int,
                          c_void_p]),
    'pgt_adain_frames': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                 c_void_p, c_int, c_void_p]),
    'pgt_maxpool3x3s2': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    'pgt_global_avgpool': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    'pgt_channel_affine': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_int,
                                   c_void_p, c_int, c_void_p, c_int, c_void_p]),
    'pgt_assemble_cond': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_void_p, c_int, c_void_p]),
    'pgt_u8hwc_to_f32nchw': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    'pgt_u8hwc_resize_to_f32nchw': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p,
                                            c_void_p]),
    'pgt_f32nchw_resize_to_f32nchw': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'pgt_imresize_u8hwc_to_f32nchw': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                              c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'pgt_f32nchw_to_u8hwc': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'pgt_gather_frames': (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_scatter_frames': (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    'pgt_frame_scores_ws_doubles': (c_int64, [c_int, c_int, c_int]),
    'pgt_frame_scores': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'pgt_copy2d': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    'pgt_regroup_frames': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    'pgt_nchw_f32_to_nhwc_bf16': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                          c_void_p]),
    'pgt_nhwc_bf16_to_f32': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
}

_lib = None


def load(build_if_missing=True):
    """Loads (building first if needed) the CUDA library; raises RuntimeError when unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        # always goes through build(): it compares the source fingerprint with lib/build.stamp, so a stale binary next
        # to a fresh checkout is rebuilt instead of silently loaded (a no-op when up to date, or without nvcc)
        from . import build as _build
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('libpgt_b200.so not built: run `python -m pgtformer_b200.build`')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise RuntimeError('libpgt_b200.so does not export %s (stale build?)' % name) from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status):
    if status != 0:
        lib = load()
        msg = lib.pgt_strerror(status).decode()
        if status == -2:
            msg += ': ' + lib.pgt_last_cuda_error().decode()
        raise RuntimeError('libpgt_b200: ' + msg)
