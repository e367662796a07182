"""CPU oracle for the gray branch of whole-image mode -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

What ``FaceRestoreHelper`` does with a gray input image, restated in numpy on top of oracle/pasteback_oracle.py:

  * ``add_restored_face`` turns every restored face into ``adain_npy(bgr2gray(restored), cropped)``: a float64 face whose three
    channels carry the restored luminance with the per-channel mean and std of the cropped input face;
  * ``paste_faces_to_input_image`` then warps float64 faces.  cv2.warpAffine on CV_64F uses the same 1/32 fixed-point
    coordinates as on uint8 but blends with the float32 weight table, products and the left-to-right sum in double; and numpy's
    promotion makes the canvas float64 from the first face on (its first ``(1 - mask) * canvas`` without a parse mask is still a
    float32 product, the canvas being uint8 then);
  * the result is ``astype(np.uint16)`` when the canvas exceeds 256 and ``astype(np.uint8)`` otherwise.

tests/test_oracle_lanczos_gray.py pins both against the reference's own functions on the CPU.
"""
import numpy as np

from . import pasteback_oracle as O


def bgr2gray(img):
    """0.2989 r + 0.5870 g + 0.1140 b in float64, repeated to three channels."""
    b, g, r = img[:, :, 0], img[:, :, 1], img[:, :, 2]
    gray = 0.2989 * r + 0.5870 * g + 0.1140 * b
    return gray[:, :, None].repeat(3, axis=2)


def mean_std(feat, eps=1e-5):
    """Per channel over all pixels: mean and sqrt(population variance + eps)."""
    flat = feat.reshape(-1, feat.shape[2]).astype(np.float64)
    return flat.mean(axis=0), np.sqrt(flat.var(axis=0) + eps)


def gray_adain(restored, cropped):
    """add_restored_face on a gray image: (gray - content mean) / content std * style std + style mean."""
    content = bgr2gray(restored)
    smean, sstd = mean_std(cropped)
    cmean, cstd = mean_std(content)
    return (content - cmean) / cstd * sstd + smean


def warp_linear_f64(face, M, dsize):
    """cv2.warpAffine(face float64 HWC, M, dsize) with the constant border 0."""
    return np.stack([O.warp_linear_float(np.ascontiguousarray(face[:, :, c]), M, dsize) for c in range(face.shape[2])], axis=2)


def paste_faces_f64(input_img, restored_faces, inverse_affines, upscale, parse_masks=None, upsample_img=None, face_size=512):
    """oracle.pasteback_oracle.paste_faces for float64 restored faces (no face upsampler: it returns uint8 faces).  Returns
    the canvas before the final cast; inverse_affines are adjusted in place as the reference does."""
    h, w = input_img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    canvas = O.resize_linear_u8(input_img, (w_up, h_up)) if upsample_img is None else upsample_img
    for i, (face, inv) in enumerate(zip(restored_faces, inverse_affines)):
        inv[:, 2] += 0.5 * upscale if upscale > 1 else 0
        inv_restored = warp_linear_f64(face, inv, (w_up, h_up))
        inv_mask = O.warp_linear_float(np.ones((face_size, face_size), np.float32), inv, (w_up, h_up))
        erosion = O.erode_rect(inv_mask, int(2 * upscale))
        pasted = erosion[:, :, None] * inv_restored                   # float32 * float64
        w_edge = int(np.sum(erosion, dtype=np.float64) ** 0.5) // 20
        center = O.erode_rect(erosion, w_edge * 2)
        m = O.blur_reflect101(center, O.gaussian_kernel(2 * w_edge + 1, 0, np.float32))[:, :, None]
        if parse_masks is not None:
            pm = O.resize_linear_f64(O.parse_soft_mask(parse_masks[i]), (face_size, face_size))
            pm = O.warp_linear_float(pm, inv, (w_up, h_up))[:, :, None]
            m = np.where(pm < m, pm, m.astype(np.float64))
        canvas = m * pasted + (1 - m) * canvas                        # numpy's promotion: see the module docstring
    return canvas


def final_cast(canvas):
    """paste_faces_to_input_image:496-499: uint16 when the canvas exceeds 256, else uint8 (truncation, low bits kept)."""
    t = np.trunc(canvas).astype(np.int64)
    return t.astype(np.uint16) if np.max(canvas) > 256 else t.astype(np.uint8)
