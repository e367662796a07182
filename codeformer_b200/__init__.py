"""codeformer_b200 -- H100-native (sm_90a) execution of CodeFormer's core forward pass.

Public surface = the reference's plugin API for this path (SURVEY.md §8b):
    ARCH_REGISTRY.get('CodeFormer') / .get('VQAutoEncoder')     basicsr/utils/registry.py:62
    CodeFormer(...).forward(x, w, detach_16, code_only, adain)  basicsr/archs/codeformer_arch.py:223
    VQAutoEncoder(...).forward(x)                               basicsr/archs/vqgan_arch.py:385
"""
from .registry import ARCH_REGISTRY, install          # noqa: F401
from .arch import CodeFormer, VQAutoEncoder, VectorQuantizer   # noqa: F401
from .upsampler import RRDBNet, RealESRGANer                   # noqa: F401
from .parsing import ParseNet, face_parse_mask, init_parsing_model   # noqa: F401
from .bisenet import BiSeNet   # noqa: F401
from .pasteback import warp_faces, paste_faces, align_warp_face, paste_faces_to_input_image   # noqa: F401
from .detection import RetinaFace, init_detection_model   # noqa: F401
from .yolov5face import YOLOv5lFace, YoloDetector   # noqa: F401
from .pasteback import resize_area, warp_faces_multi, paste_faces_multi   # noqa: F401
from .pasteback import resize_lanczos4, gray_adain_faces, add_restored_face   # noqa: F401
from .wholeimage import restore_images, restore_images_sweep, restore_aligned   # noqa: F401
from .arcface import ResNetArcFace, identity_similarity   # noqa: F401
from .metrics import calculate_psnr, calculate_ssim, psnr_ssim   # noqa: F401
from .lpips import LPIPS, LPIPSLoss, lpips_distance   # noqa: F401
from .degradation import degrade_faces, sample_degradations, jpeg_roundtrip   # noqa: F401
from .fid import (InceptionV3, inception_features, fid_statistics, frechet_distance, calculate_fid,   # noqa: F401
                  fid_scores)


def check_async_status():
    """Raise ``RuntimeError`` if a kernel of an earlier (asynchronous) forward on the current device reported a failure --
    a tensor-core pipeline time-out or an activation outside the fp16 operand range.  Call after synchronising the stream;
    the next forward and the ``restore_faces`` / ``forward_host`` front-ends check by themselves (include/cfb200.h)."""
    from . import _lib
    _lib.check(_lib.load().cfb_check_async_status(), 'check_async_status')


__all__ = ['ARCH_REGISTRY', 'install', 'CodeFormer', 'VQAutoEncoder', 'VectorQuantizer', 'RRDBNet', 'RealESRGANer', 'ParseNet', 'BiSeNet', 'face_parse_mask', 'init_parsing_model',
           'warp_faces', 'paste_faces', 'align_warp_face', 'paste_faces_to_input_image', 'RetinaFace', 'init_detection_model',
           'YOLOv5lFace', 'YoloDetector', 'resize_area', 'warp_faces_multi', 'paste_faces_multi', 'restore_images',
           'resize_lanczos4', 'gray_adain_faces', 'add_restored_face', 'restore_aligned', 'restore_images_sweep',
           'ResNetArcFace', 'identity_similarity', 'calculate_psnr', 'calculate_ssim', 'psnr_ssim', 'LPIPS', 'LPIPSLoss', 'lpips_distance',
           'degrade_faces', 'sample_degradations', 'jpeg_roundtrip', 'InceptionV3', 'inception_features', 'fid_statistics',
           'frechet_distance', 'calculate_fid', 'fid_scores',
           'check_async_status']
