"""ctypes binding of libcfb200.so (the C ABI declared in include/cfb200.h).

The product path has NO fallback: if the shared library is missing or cannot be loaded this
module raises, and every forward raises ``RuntimeError(cfb_last_error())`` on a non-zero status
(callers of the reference catch exceptions and fall back to the input face,
/root/reference/inference_codeformer.py:209-211 -- so errors must be exceptions, never aborts).
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libcfb200.so')


class CfbConfig(Structure):
    _fields_ = [('kind', c_int32), ('img_size', c_int32), ('nf', c_int32), ('n_ch_mult', c_int32),
                ('ch_mult', c_int32 * 8), ('res_blocks', c_int32), ('n_attn_res', c_int32),
                ('attn_res', c_int32 * 4), ('codebook_size', c_int32), ('emb_dim', c_int32), ('beta', c_float),
                ('dim_embd', c_int32), ('n_head', c_int32), ('n_layers', c_int32), ('latent_size', c_int32),
                ('n_connect', c_int32), ('connect', c_int32 * 6)]


_P = c_void_p
# name -> (restype, argtypes); every symbol include/cfb200.h declares
SIGNATURES = {
    'cfb_version': (c_int, []),
    'cfb_last_error': (c_char_p, []),
    'cfb_device_info': (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    'cfb_net_create': (c_void_p, [POINTER(CfbConfig)]),
    'cfb_net_destroy': (None, [_P]),
    'cfb_net_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_net_prepare': (c_int, [_P, _P]),
    'cfb_workspace_bytes': (c_int64, [_P, c_int32]),
    'cfb_last_launch_count': (c_int64, [_P]),
    'cfb_net_set_engine': (c_int, [_P, c_int32]),
    'cfb_net_set_precision': (c_int, [_P, c_int32]),
    'cfb_net_capture': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_codeformer_forward': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_float, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_host_io_bytes': (c_int64, [_P, c_int32]),
    'cfb_codeformer_forward_host': (c_int, [_P, _P, _P, _P, _P, c_int32, c_float, c_int32, _P, c_int64, _P, c_int64, _P]),
    'cfb_codeformer_forward_u8': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_float, c_int32, _P, c_int64, _P]),
    'cfb_codeformer_inpaint_u8': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_float, c_int32, _P, c_int64, _P]),
    'cfb_codeformer_forward_wv': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, _P, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_codeformer_forward_u8_wv': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, _P, c_int32, _P, c_int64, _P]),
    'cfb_codeformer_inpaint_u8_wv': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, _P, c_int32, _P, c_int64, _P]),
    'cfb_sweep_workspace_bytes': (c_int64, [_P, c_int32, c_int32]),
    'cfb_codeformer_sweep_u8': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_int32, _P, c_int32, _P, c_int64, _P]),
    'cfb_codeformer_restore_host': (c_int, [_P, _P, _P, c_int32, c_float, c_int32, _P, c_int64, _P, c_int64, _P]),
    'cfb_u8_to_input': (c_int, [_P, _P, c_int32, c_int32, _P]),
    'cfb_output_to_u8': (c_int, [_P, _P, c_int32, c_int32, _P]),
    'cfb_vqae_forward': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, _P, c_int64, _P]),
    'cfb_vq_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32, c_int32]),
    'cfb_vq_nearest': (c_int, [_P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_float, _P, _P, _P, _P, _P, c_int64, _P]),
    'cfb_vq_fast_supported': (c_int32, [c_int32] * 5),
    'cfb_vq_prepared_bytes': (c_int64, [c_int32, c_int32]),
    'cfb_vq_prepare': (c_int, [_P, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_vq_fast_workspace_bytes': (c_int64, [c_int32] * 4),
    'cfb_vq_nearest_fast': (c_int, [_P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_float, _P, _P, _P, _P, _P, c_int64, _P]),
    'cfb_codebook_lookup': (c_int, [_P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, _P, _P]),
    'cfb_conv2d_nhwc': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                _P, _P, c_int32, _P, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_conv2d_workspace_bytes': (c_int64, [c_int32] * 7),
    'cfb_gn_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32]),
    'cfb_group_norm_coef': (c_int, [_P, _P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_float, _P, c_int64, _P]),
    'cfb_affine_act': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_attention': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_float, _P]),
    'cfb_layer_norm': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_adain_nhwc': (c_int, [_P, _P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_debug_time_conv': (c_int, [_P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P, c_int64,
                                   _P, _P, _P, c_int32, POINTER(c_float)]),
    'cfb_debug_conv_tc': (c_int, [_P, _P, c_int32, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                 _P, _P, c_int32, _P, _P, _P, c_float, _P, _P, _P, c_int64, _P, POINTER(c_int32)]),
    'cfb_debug_conv_tc_prec': (c_int, [_P, _P, c_int32, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                      _P, _P, c_int32, _P, _P, _P, c_float, _P, _P, _P, c_int64, _P, POINTER(c_int32), c_int32,
                                      c_int32, c_int32]),
    'cfb_debug_conv_tc_prec_wv': (c_int, [_P, _P, c_int32, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                         _P, _P, c_int32, _P, _P, _P, _P, _P, _P, _P, c_int64, _P, POINTER(c_int32), c_int32,
                                         c_int32, c_int32]),
    'cfb_debug_bmm_tc_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32]),
    'cfb_debug_bmm_tc': (c_int, [_P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_debug_layer_norm_planes': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_debug_code_lookup': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_debug_gn_partials_workspace_bytes': (c_int64, [c_int32, c_int32]),
    'cfb_debug_gn_coef_from_partials': (c_int, [_P, c_int32, _P, _P, _P, _P, c_int32, c_int32, c_int32, c_float, _P, c_int64, _P]),
    'cfb_debug_gn_cat_partials': (c_int, [_P, _P, _P, c_int64, c_int32, _P]),
    'cfb_rrdb_create': (c_void_p, [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32]),
    'cfb_rrdb_destroy': (None, [_P]),
    'cfb_rrdb_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_rrdb_prepare': (c_int, [_P, _P]),
    'cfb_rrdb_set_precision': (c_int, [_P, c_int32]),
    'cfb_rrdb_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32]),
    'cfb_rrdb_forward': (c_int, [_P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_rrdb_forward_u8_tiles': (c_int, [_P, _P, c_int32, c_int32, c_int32, c_int32, _P, c_int32, c_int32, c_int32, _P, _P,
                                          c_int64, _P]),
    'cfb_rrdb_forward_tiles': (c_int, [_P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, _P, c_int32, c_int32, c_int32, _P,
                                       c_int32, _P, _P, c_int64, _P]),
    'cfb_parsenet_create': (c_void_p, [c_int32] * 8),
    'cfb_parsenet_destroy': (None, [_P]),
    'cfb_parsenet_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_parsenet_prepare': (c_int, [_P, _P]),
    'cfb_parsenet_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32]),
    'cfb_parsenet_forward': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_parse_argmax': (c_int, [_P, _P, _P, c_int32, c_int32, c_int64, _P]),
    'cfb_parsenet_set_precision': (c_int, [_P, c_int32]),
    'cfb_parsenet_masks_u8': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_conv2d_gen_workspace_bytes': (c_int64, [c_int32, c_int32]),
    'cfb_conv2d_gen_nhwc': (c_int, [_P, c_int32, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                    c_int32, c_int32, c_int32, _P, c_int32, _P, c_int32, c_float, _P, c_int64, _P]),
    'cfb_conv2d_gen_nhwc_prec': (c_int, [_P, c_int32, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                         c_int32, c_int32, c_int32, c_int32, _P, c_int32, _P, c_int32, c_float, _P, c_int64, _P,
                                         c_int32]),
    'cfb_conv2d_pertap_workspace_bytes': (c_int64, [c_int32] * 7),
    'cfb_conv2d_pertap_nhwc': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P,
                                       _P, c_int64, _P]),
    'cfb_conv2d_pertap_slice_nhwc': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                             c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_retinaface_priors': (c_int64, [c_int32, c_int32]),
    'cfb_retinaface_create': (c_void_p, []),
    'cfb_retinaface_destroy': (None, [_P]),
    'cfb_retinaface_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_retinaface_prepare': (c_int, [_P, _P]),
    'cfb_retinaface_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32]),
    'cfb_retinaface_forward': (c_int, [_P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_retinaface_forward_u8': (c_int, [_P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_retinaface_candidates': (c_int, [_P, _P, _P, c_int32, c_int32, c_int32, c_float, _P, _P, _P]),
    'cfb_bisenet_create': (c_void_p, [c_int32]),
    'cfb_bisenet_destroy': (None, [_P]),
    'cfb_bisenet_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_bisenet_prepare': (c_int, [_P, _P]),
    'cfb_bisenet_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32]),
    'cfb_bisenet_forward': (c_int, [_P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_bisenet_masks_u8': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_debug_bisenet_bilinear': (c_int, [_P, c_int32, c_int32, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P]),
    'cfb_debug_bisenet_attention': (c_int, [_P, c_int32, c_int32, c_int32, _P, _P, c_int32, c_int32, _P, _P, c_int32, c_int32, _P, _P,
                                            _P]),
    'cfb_arcface_create': (c_void_p, [c_int32, c_int32, c_int32, c_int32]),
    'cfb_arcface_destroy': (None, [_P]),
    'cfb_arcface_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_arcface_prepare': (c_int, [_P, _P]),
    'cfb_arcface_workspace_bytes': (c_int64, [_P, c_int32]),
    'cfb_arcface_forward': (c_int, [_P, _P, _P, c_int32, _P, c_int64, _P]),
    'cfb_arcface_forward_u8': (c_int, [_P, _P, _P, c_int32, _P, c_int64, _P]),
    'cfb_debug_arcface_conv': (c_int, [_P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P, _P, c_int32,
                                       c_float, _P, _P, c_int64, _P]),
    'cfb_yolov5face_predictions': (c_int64, [c_int32, c_int32]),
    'cfb_yolov5face_create': (c_void_p, []),
    'cfb_yolov5face_destroy': (None, [_P]),
    'cfb_yolov5face_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_yolov5face_prepare': (c_int, [_P, _P]),
    'cfb_yolov5face_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32]),
    'cfb_yolov5face_forward': (c_int, [_P, _P, _P, _P, _P, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    'cfb_yolov5face_forward_u8': (c_int, [_P, _P, c_int32, c_int32, c_int32, c_int32, _P, _P, _P, _P, c_int32, c_int32, c_int32,
                                          _P, c_int64, _P]),
    'cfb_yolov5face_candidates': (c_int, [_P, c_int32, c_int32, c_int32, c_float, _P, _P, _P]),
    'cfb_lpips_create': (c_void_p, []),
    'cfb_lpips_destroy': (None, [_P]),
    'cfb_lpips_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_lpips_prepare': (c_int, [_P, _P]),
    'cfb_lpips_workspace_bytes': (c_int64, [_P, c_int32, c_int32, c_int32, c_int32]),
    'cfb_lpips_forward': (c_int, [_P, _P, _P] + [c_int32] * 5 + [_P, _P, _P, c_int64, _P]),
    'cfb_lpips_forward_u8': (c_int, [_P, _P, _P] + [c_int32] * 5 + [_P, _P, _P, c_int64, _P]),
    'cfb_lpips_u8_table': (c_int, [c_int32, _P, _P, _P]),
    'cfb_debug_lpips_stem': (c_int, [_P, _P, _P, c_int32, c_int32, _P, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_debug_lpips_head_workspace_bytes': (c_int64, [c_int32] * 4),
    'cfb_debug_lpips_head': (c_int, [_P, _P, _P, _P] + [c_int32] * 5 + [_P, c_int64, _P]),
    'cfb_fid_create': (c_void_p, []),
    'cfb_fid_destroy': (None, [_P]),
    'cfb_fid_set_param': (c_int, [_P, c_char_p, _P, c_int64]),
    'cfb_fid_prepare': (c_int, [_P, _P]),
    'cfb_fid_workspace_bytes': (c_int64, [_P] + [c_int32] * 4),
    'cfb_fid_forward': (c_int, [_P, _P] + [c_int32] * 5 + [_P, _P, c_int64, _P]),
    'cfb_fid_forward_u8': (c_int, [_P, _P] + [c_int32] * 3 + [_P, _P, c_int64, _P]),
    'cfb_fid_input': (c_int, [_P] + [c_int32] * 6 + [_P, _P]),
    'cfb_fid_stats': (c_int, [_P, c_int64, c_int32, _P, _P, _P]),
    'cfb_debug_fid_pool': (c_int, [_P, _P] + [c_int32] * 5 + [_P]),
    'cfb_conv2d_pertap_window_workspace_bytes': (c_int64, [c_int32] * 10),
    'cfb_conv2d_pertap_window_nhwc': (c_int, [_P, _P, _P, _P] + [c_int32] * 13 + [_P, c_int64, _P]),
    'cfb_psnr_ssim_workspace_bytes': (c_int64, [c_int32] * 6),
    'cfb_psnr_ssim': (c_int, [_P, _P] + [c_int32] * 10 + [_P, _P, _P, c_int64, _P]),
    'cfb_degrade_workspace_bytes': (c_int64, [c_int32, c_int32, _P, _P]),
    'cfb_degrade_faces': (c_int, [_P, c_int32, c_int32, _P, c_int32, _P, _P, _P, _P, c_int32, _P, _P, c_int64, _P]),
    'cfb_debug_degrade_faces': (c_int, [_P, c_int32, c_int32, _P, c_int32, _P, _P, _P, _P, c_int32, _P, _P, c_int64, _P, _P, _P]),
    'cfb_degrade_color_workspace_bytes': (c_int64, [c_int32, c_int32, _P, _P, _P, c_int32]),
    'cfb_degrade_faces_color': (c_int, [_P, c_int32, c_int32, _P, c_int32, _P, _P, _P, _P, _P, _P, _P, c_int32, _P, _P, c_int64,
                                        _P]),
    'cfb_debug_degrade_faces_color': (c_int, [_P, c_int32, c_int32, _P, c_int32, _P, _P, _P, _P, _P, _P, _P, c_int32, _P, _P,
                                              c_int64, _P, _P]),
    'cfb_jpeg_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32]),
    'cfb_jpeg_roundtrip': (c_int, [_P, _P, c_int32, c_int32, c_int32, _P, _P, c_int64, _P]),
    'cfb_check_async_status': (c_int, []),
    'cfb_debug_set_wait_limit': (c_int, [c_int64]),
    'cfb_debug_inject_fault': (c_int, [c_int32]),
    'cfb_debug_set_stamps': (c_int, [_P]),
    'cfb_nchw_to_nhwc': (c_int, [_P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_nhwc_to_nchw': (c_int, [_P, _P, c_int32, c_int32, c_int32, _P]),
    'cfb_warp_affine_u8': (c_int, [_P, c_int32, c_int32, _P, c_int32, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_resize_linear_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P]),
    'cfb_paste_faces_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_paste_faces': (c_int, [_P, c_int32, c_int32, _P, c_int32, c_int32, _P, _P, c_double, _P, _P, _P, c_int64, _P]),
    'cfb_resize_area_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P]),
    'cfb_resize_linear_scale_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, c_double, c_double, _P]),
    'cfb_warp_affine_multi_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, _P, c_int32, _P, c_int32, c_int32, c_int32, c_int32,
                                         c_int32, c_int32, _P]),
    'cfb_paste_faces_multi_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_paste_faces_multi': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P, _P, _P, c_double, _P, _P, c_int64, _P]),
    'cfb_resize_lanczos4_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P]),
    'cfb_lanczos4_table': (None, [c_int32, c_int32, _P, _P]),
    'cfb_resize_lanczos4_u16': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P]),
    'cfb_lanczos4_table_f32': (None, [c_int32, c_int32, _P, _P]),
    'cfb_gray_adain_faces': (c_int, [_P, _P, c_int32, c_int32, _P, _P, _P]),
    'cfb_is_gray_u8': (c_int, [_P, c_int32, c_int32, c_int32, _P, _P]),
    'cfb_f64_to_input': (c_int, [_P, _P, c_int32, c_int32, _P]),
    'cfb_paste_faces_f64_workspace_bytes': (c_int64, [c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, _P]),
    'cfb_paste_faces_f64': (c_int, [_P, c_int32, c_int32, c_int32, _P, c_int32, c_int32, _P, _P, _P, c_double, _P, _P, _P, _P,
                                    c_int64, _P]),
}

_lib = None


def load():
    """Load libcfb200.so (built in-tree by ``codeformer_b200/build.py`` / ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        # a fresh checkout has no binary: compile the CUDA sources in-tree (nvcc, sm_90a).  Never a CPU/PyTorch fallback:
        # if that is impossible the import fails loudly.  build() serialises concurrent importers (torchrun ranks, xdist
        # workers) on a file lock and publishes the library with an atomic rename.
        try:
            from . import build as _build
            _build.build(force=False)
        except Exception as e:  # noqa: BLE001
            raise RuntimeError(f'{LIB_PATH} is missing and could not be built with nvcc ({e}); there is no CPU or '
                               'PyTorch fallback for this path -- run `python -m codeformer_b200.build`') from e
    # CFB_LIB: load another build of the SAME library (A/B timing of two kernel versions in one process);
    # only there may a diagnostics entry point (cfb_debug_*) be absent from an older build
    override = os.environ.get('CFB_LIB')
    lib = ctypes.CDLL(override if override else LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        if override and name.startswith('cfb_debug_') and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)            # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.cfb_version() != 100:
        raise RuntimeError('libcfb200.so version mismatch')
    _lib = lib
    return lib


def check(status, what=''):
    if status != 0:
        msg = load().cfb_last_error()
        raise RuntimeError(f'libcfb200 {what} failed: {msg.decode() if msg else "unknown error"}')


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream(device=None):
    """The current CUDA stream of ``device`` (default: the current device), as the ``void* stream`` argument."""
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
