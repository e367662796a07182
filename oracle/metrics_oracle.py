"""PSNR and SSIM as basicsr computes them (basicsr/metrics/psnr_ssim.py, metric_util.py, bgr2ycbcr of
utils/matlab_functions.py), restated in numpy / cv2 for the tests of codeformer_b200.metrics.

The contract, with the package's deliberate deviations from the reference:
  * equal shapes; input_order 'HWC' or 'CHW' (ValueError otherwise); a 2-D image is one channel;
  * uint8, uint16, float32 or float64 only (NotImplementedError otherwise); the two images may differ in dtype;
  * crop_border pixels dropped from each edge; a negative crop_border, or a cropped image with no pixels (PSNR) or a side
    under 11 (SSIM), raises ValueError -- the reference returns NaN with a warning or fails inside cv2 there;
  * test_y_channel: v = float32(x) / 255 in float32; for three channels Y = (c0 * 24.966 + c1 * 128.553) + c2 * 65.481 + 16
    in float64 (channel 0 is blue), / 255 rounded to float32; other channel counts keep v; then * 255 in float32;
  * PSNR: mse = mean((a - b)^2) over every value, inf when mse == 0, else 20 log10(255 / sqrt(mse)) -- peak 255 for every
    dtype.  On the Y path the squared differences are float32, as in the reference, but their mean is taken in float64
    (the reference's float32 mean differs from it by up to about 1e-5 dB);
  * SSIM, per channel: the five float64 maps filtered with the outer product of cv2.getGaussianKernel(11, 1.5), valid
    region only, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2, the map's mean; then the mean over the channels.
"""
import cv2
import numpy as np

DTYPES = (np.uint8, np.uint16, np.float32, np.float64)
SSIM_MIN_SIDE = 11


def prepare(img1, img2, crop_border, input_order='HWC', test_y_channel=False, min_side=1):
    """The cropped images the metrics are computed on: float64 HWC, or float32 HWC on the Y path."""
    assert img1.shape == img2.shape, f'Image shapes differ: {img1.shape}, {img2.shape}.'
    if input_order not in ('HWC', 'CHW'):
        raise ValueError(f'Wrong input_order {input_order}. Supported input_orders are "HWC" and "CHW"')
    if crop_border < 0:
        raise ValueError(f'crop_border must be >= 0, got {crop_border}')
    out = []
    for img in (img1, img2):
        if img.dtype not in DTYPES:
            raise NotImplementedError(f'dtype {img.dtype} is not supported (uint8, uint16, float32, float64)')
        if img.ndim == 2:
            img = img[..., None]
        elif input_order == 'CHW':
            img = img.transpose(1, 2, 0)
        h, w = img.shape[:2]
        if h - 2 * crop_border < min_side or w - 2 * crop_border < min_side:
            raise ValueError(f'{h}x{w} image with crop_border {crop_border} leaves less than {min_side} pixel(s) per side')
        img = img[crop_border:h - crop_border, crop_border:w - crop_border].astype(np.float64)
        out.append(y_channel(img) if test_y_channel else img)
    return out


def y_channel(img):
    """Y of an HWC float64 image whose values are those of the input dtype (float32 [H,W,1]); other channel counts
    than three keep their channels, rounded through float32(x) / 255 * 255."""
    v = img.astype(np.float32) / np.float32(255)
    if img.shape[2] == 3:
        v64 = v.astype(np.float64)
        y = v64[..., 0] * 24.966 + v64[..., 1] * 128.553
        y = y + v64[..., 2] * 65.481
        y = y + 16.0
        v = (y / 255.).astype(np.float32)[..., None]
    return v * np.float32(255)


def psnr(img1, img2, crop_border, input_order='HWC', test_y_channel=False):
    a, b = prepare(img1, img2, crop_border, input_order, test_y_channel)
    sq = (a - b) ** 2
    mse = np.sum(sq.astype(np.float64)) / sq.size if test_y_channel else np.mean(sq)
    if mse == 0:
        return float('inf')
    return 20. * np.log10(255. / np.sqrt(mse))


def gaussian_window():
    g = cv2.getGaussianKernel(11, 1.5)
    return g @ g.T


def ssim_channel(a, b):
    """Mean SSIM map of two float64 single-channel images (valid region of the 11 x 11 window)."""
    win = gaussian_window()
    c1, c2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2

    def blur(x):
        return cv2.filter2D(x, -1, win)[5:-5, 5:-5]
    mu_a, mu_b = blur(a), blur(b)
    aa, bb, ab = mu_a ** 2, mu_b ** 2, mu_a * mu_b
    var_a, var_b, cov = blur(a ** 2) - aa, blur(b ** 2) - bb, blur(a * b) - ab
    return (((2 * ab + c1) * (2 * cov + c2)) / ((aa + bb + c1) * (var_a + var_b + c2))).mean()


def ssim(img1, img2, crop_border, input_order='HWC', test_y_channel=False):
    a, b = prepare(img1, img2, crop_border, input_order, test_y_channel, min_side=SSIM_MIN_SIDE)
    a, b = a.astype(np.float64), b.astype(np.float64)
    return np.array([ssim_channel(a[..., i], b[..., i]) for i in range(a.shape[2])]).mean()
