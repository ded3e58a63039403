"""ctypes binding of libocc_b200.so (include/occ_b200.h).  There is no CPU fallback: if the
library is missing or a call fails, an exception is raised."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libocc_b200.so')

c_f32p = ctypes.c_void_p
_vp = ctypes.c_void_p
_i = ctypes.c_int
_i64 = ctypes.c_int64
_f64 = ctypes.c_double


class OccConfig(ctypes.Structure):
    _fields_ = [('bev_h', _i), ('bev_w', _i), ('embed_dims', _i), ('num_heads', _i), ('num_layers', _i),
                ('num_cams', _i), ('num_levels', _i), ('level_h', _i * 4), ('level_w', _i * 4),
                ('num_points_in_pillar', _i), ('sca_points', _i), ('tsa_points', _i), ('ffn_dim', _i),
                ('pillar_h', _i), ('out_dim', _i), ('num_classes', _i), ('pc_range', ctypes.c_float * 6),
                ('precision', _i), ('use_tensor_cores', _i), ('use_cams_embeds', _i),
                ('rotate_center', _i * 2)]


# name -> (restype, argtypes); every symbol declared in include/occ_b200.h
SIGNATURES = {
    'occb200_last_error': (ctypes.c_char_p, []),
    'occb200_version': (ctypes.c_char_p, []),
    'occb200_ms_deform_attn_forward': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    'occb200_ms_deform_attn_backward': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'occb200_engine_create': (_i, [ctypes.POINTER(OccConfig), ctypes.POINTER(_vp)]),
    'occb200_engine_destroy': (None, [_vp]),
    'occb200_engine_load_param': (_i, [_vp, ctypes.c_char_p, _vp, _i64]),
    'occb200_engine_finalize': (_i, [_vp]),
    'occb200_engine_set_cameras': (_i, [_vp, _vp, _vp, _i, _i]),
    'occb200_engine_set_input_dtype': (_i, [_vp, _i]),
    'occb200_engine_attach_backbone': (_i, [_vp, _vp]),
    'occb200_engine_set_prev_rotation': (_i, [_vp, _vp]),
    'occb200_engine_set_prev_rotation_angle': (_i, [_vp, _f64]),
    'occb200_rotation_coeffs': (_i, [_f64, _i, _i, _i, _i, _vp]),
    'occb200_engine_rotation_map': (_i, [_vp, _f64, _vp, _vp]),
    'occb200_engine_forward': (_i, [_vp, ctypes.POINTER(_vp), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'occb200_engine_forward_host': (_i, [_vp, ctypes.POINTER(_vp), _vp, _vp, _vp]),
    'occb200_engine_submit_host': (_i, [_vp, _i, ctypes.POINTER(_vp), _vp, _vp, _vp]),
    'occb200_engine_wait_host': (_i, [_vp, _i]),
    'occb200_engine_set_history': (_i, [_vp, _i]),
    'occb200_engine_forward_video': (_i, [_vp, ctypes.POINTER(_vp), _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    'occb200_engine_submit_host_video': (_i, [_vp, _i, ctypes.POINTER(_vp), _vp, _i, _vp, _vp, _vp]),
    'occb200_engine_forward_video_angle': (_i, [_vp, ctypes.POINTER(_vp), _f64, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    'occb200_engine_submit_host_video_angle': (_i, [_vp, _i, ctypes.POINTER(_vp), _f64, _i, _vp, _vp, _vp]),
    'occb200_engine_set_rays': (_i, [_vp, _vp, _i]),
    'occb200_engine_request_rays': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    'occb200_engine_request_score': (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    'occb200_ray_score': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp]),
    'occb200_ray_records': (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    'occb200_engine_enable_taps': (_i, [_vp, _i]),
    'occb200_engine_copy_tap': (_i, [_vp, _i, _i, _vp, _vp]),
    'occb200_engine_project_pillars': (_i, [_vp, _vp, _vp, _vp]),
    'occb200_engine_launches_per_frame': (_i, [_vp]),
    'occb200_engine_profile': (_i, [_vp, _i]),
    'occb200_engine_profile_read': (_i, [_vp, _vp, _vp, _i]),
    'occb200_render_forward': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i64, _vp, _vp, _vp, _vp]),
    'occb200_ray_metric_accumulate': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    'occb200_linear_f32': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    'occb200_layernorm_f32': (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    'occb200_gemm_bf16_tc': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'occb200_gemm_tc': (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'occb200_gemm_tc_ln': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    'occb200_gemm_tc_blocked256': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'occb200_gemm_tc_tsa_inputs': (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'occb200_gemm_tc_split3': (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'occb200_split_bf16': (_i, [_vp, _i, _vp, _i, _i64, _vp, _vp]),
    'occb200_tsa_gather': (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _vp, _vp]),
    'occb200_sca_gather': (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'occb200_decoder_lift': (_i, [_i, _i, _i, _vp, _i, _i, _vp, ctypes.POINTER(_i), _vp]),
    'occb200_decoder_conv3d': (_i, [_i, _i, _vp, _i, _i, _i, _vp, _vp, _vp, ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    'occb200_decoder_head': (_i, [_i, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    'occb200_encoder_dense': (_i, [_i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, ctypes.POINTER(_i),
                                   ctypes.POINTER(_i), _vp]),
    'occb200_encoder_layernorm': (_i, [_i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    'occb200_encoder_pack': (_i, [_i, _i, ctypes.POINTER(_vp), _i, _vp, _i, _vp, _vp, _vp, _vp]),
    'occb200_encoder_prepare_query': (_i, [_i, _i, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    'occb200_t32_convert': (_i, [_vp, _vp, _i64, _i, _i, _vp]),
    'occb200_backbone_create': (_vp, [_i, _i, _i, _i, _i]),
    'occb200_backbone_destroy': (None, [_vp]),
    'occb200_backbone_load_param': (_i, [_vp, ctypes.c_char_p, _vp, ctypes.c_int64]),
    'occb200_backbone_finalize': (_i, [_vp]),
    'occb200_backbone_level_shape': (_i, [_vp, _i, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    'occb200_backbone_forward': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'occb200_backbone_forward_nhwc_bf16': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'occb200_backbone_set_frame_format': (_i, [_vp, _i, _i, _vp, _vp, _i]),
    'occb200_backbone_forward_frames': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    'occb200_backbone_conv': (_i, [_i, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp,
                                   ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    'occb200_backbone_maxpool': (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp]),
    'occb200_backbone_upsample_add': (_i, [_i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    'occb200_jpeg_create': (_i, [ctypes.POINTER(_vp)]),
    'occb200_jpeg_destroy': (None, [_vp]),
    'occb200_jpeg_info': (_i, [_vp, _i64, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    'occb200_jpeg_decode': (_i, [_vp, _i, _vp, _vp, _vp, _i64, _vp]),
    'occb200_jpeg_status': (_i, [_vp, ctypes.POINTER(_i)]),
    'occb200_engine_jpeg_status': (_i, [_vp, ctypes.POINTER(_i)]),
}


class EncodedFrame(ctypes.Structure):
    """occb200_encoded_frame: the host buffers of one frame's camera files (input dtype 4)"""
    _fields_ = [('data', _vp * 8), ('size', _i64 * 8)]

_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} is missing: run `python -m occnet_b200.build` '
                               '(libocc_b200 has no CPU / PyTorch fallback)')
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


class OccB200Error(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise OccB200Error(f'libocc_b200 error {rc}: {load().occb200_last_error().decode()}')


def ptr(t):
    """device / host pointer of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, 'data_ptr'):
        return ctypes.c_void_p(t.data_ptr())
    return ctypes.c_void_p(t.ctypes.data)


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
