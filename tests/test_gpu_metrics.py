"""-m gpu: restoration metrics on the device (codeformer_b200.metrics, cfb_psnr_ssim) against the numpy / cv2 restatement of
basicsr's calculate_psnr / calculate_ssim (oracle/metrics_oracle.py): drop-ins, batches, fidelity sweeps and lists of whole
images, determinism and the deliberate errors."""
import os

import cv2
import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import pasteback as PB
from codeformer_b200 import spec as S
from oracle import metrics_oracle as MO
from tests.test_gpu_lanczos_gray import _paste_inputs, _to_gray
from tests.test_gpu_wholeimage import nets, whole_images   # noqa: F401  (nets: fixture)
from tests.test_oracle_metrics import DTYPES, pair

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
torch.set_grad_enabled(False)
PSNR_INT_BAR = 1e-12     # integer images, batched form: the device log10 of the exact MSE
PSNR_BAR = 1e-9          # float images: float64 sums in another order
PSNR_Y_BAR = 1e-4        # Y path
SSIM_BAR = 1e-10         # separable float64 filter against cv2's


def _is_int(dtype):
    return np.dtype(dtype).kind == 'u'


def check_psnr(got, want, dtype, y, drop_in):
    if want == float('inf'):
        assert got == float('inf')
    elif _is_int(dtype) and not y and drop_in:
        assert got == want, (got, want)
    else:
        bar = PSNR_Y_BAR if y else (PSNR_INT_BAR if _is_int(dtype) else PSNR_BAR)
        assert abs(float(got) - float(want)) <= bar, (got, want)


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


@pytest.mark.parametrize('size', [(37, 50), (512, 512)], ids=['37x50', '512'])
@pytest.mark.parametrize('crop', [0, 4, 10])
@pytest.mark.parametrize('y', [False, True], ids=['rgb', 'y'])
@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
def test_drop_in_against_oracle(dtype, y, crop, size):
    a, b = pair(dtype, *size, seed=crop + 3 * y)
    ia, ib = (a, b) if crop != 4 else (_dev(a), _dev(b))      # numpy arrays and CUDA tensors
    check_psnr(cb.calculate_psnr(ia, ib, crop, test_y_channel=y), MO.psnr(a, b, crop, 'HWC', y), dtype, y, True)
    assert abs(cb.calculate_ssim(ia, ib, crop, test_y_channel=y) - MO.ssim(a, b, crop, 'HWC', y)) <= SSIM_BAR
    p, s = cb.psnr_ssim(_dev(a)[None], _dev(b)[None], crop, y)
    check_psnr(float(p[0]), MO.psnr(a, b, crop, 'HWC', y), dtype, y, False)
    assert abs(float(s[0]) - MO.ssim(a, b, crop, 'HWC', y)) <= SSIM_BAR


@pytest.mark.parametrize('y', [False, True], ids=['rgb', 'y'])
def test_chw_and_2d(y):
    a, b = pair(np.uint8, 40, 45, seed=11)
    ca, cbb = a.transpose(2, 0, 1), b.transpose(2, 0, 1)
    want_p, want_s = MO.psnr(ca, cbb, 2, 'CHW', y), MO.ssim(ca, cbb, 2, 'CHW', y)
    for ia, ib in ((ca, cbb), (_dev(ca), _dev(cbb))):
        assert cb.calculate_psnr(ia, ib, 2, 'CHW', y) == want_p
        assert abs(cb.calculate_ssim(ia, ib, 2, 'CHW', y) - want_s) <= SSIM_BAR
    for dtype in (np.uint8, np.float32):
        g, h = pair(dtype, 33, 29, c=0, seed=12)
        check_psnr(cb.calculate_psnr(g, h, 1, test_y_channel=y), MO.psnr(g, h, 1, 'HWC', y), dtype, y, True)
        assert abs(cb.calculate_ssim(_dev(g), _dev(h), 1, test_y_channel=y) - MO.ssim(g, h, 1, 'HWC', y)) <= SSIM_BAR


def test_eleven_pixel_minimum():
    for (h, w, crop) in ((11, 11, 0), (21, 30, 5), (11, 64, 0)):
        a, b = pair(np.float64, h, w, seed=h + w)
        assert abs(cb.calculate_ssim(a, b, crop) - MO.ssim(a, b, crop)) <= SSIM_BAR
        check_psnr(cb.calculate_psnr(a, b, crop), MO.psnr(a, b, crop), np.float64, False, True)
    a, b = pair(np.uint8, 20, 20, seed=1)
    with pytest.raises(ValueError):
        cb.calculate_ssim(a, b, 5)
    assert np.isfinite(cb.calculate_psnr(a, b, 9))
    with pytest.raises(ValueError):
        cb.calculate_psnr(a, b, 10)


def test_large_pair():
    a, b = pair(np.uint8, 2160, 3840, seed=21)
    for y in (False, True):
        want_p, want_s = MO.psnr(a, b, 4, 'HWC', y), MO.ssim(a, b, 4, 'HWC', y)
        check_psnr(cb.calculate_psnr(a, b, 4, test_y_channel=y), want_p, np.uint8, y, True)
        p, s = cb.psnr_ssim(_dev(a)[None], _dev(b)[None], 4, y)
        check_psnr(float(p[0]), want_p, np.uint8, y, False)
        assert abs(float(s[0]) - want_s) <= SSIM_BAR
        print(f'2160x3840 y={y}: psnr {float(p[0]):.12f} / {want_p:.12f}, ssim {float(s[0]):.15f} / {want_s:.15f}')


def _faces_pair(n, seed):
    ab = [pair(np.uint8, 512, 512, seed=seed + i) for i in range(n)]
    return np.stack([x for x, _ in ab]), np.stack([x for _, x in ab])


@pytest.mark.parametrize('B', [1, 3, 32])
def test_batched_faces(B):
    a, b = _faces_pair(B, 100)
    for y in (False, True):
        p, s = cb.psnr_ssim(_dev(a), _dev(b), 0, y)
        assert p.shape == s.shape == (B,) and p.dtype == s.dtype == torch.float64
        for i in range(min(B, 3)):
            check_psnr(float(p[i]), MO.psnr(a[i], b[i], 0, 'HWC', y), np.uint8, y, False)
            assert abs(float(s[i]) - MO.ssim(a[i], b[i], 0, 'HWC', y)) <= SSIM_BAR
        # batch invariance: every pair alone gives the same bits
        for i in range(B):
            p1, s1 = cb.psnr_ssim(_dev(a[i:i + 1]), _dev(b[i:i + 1]), 0, y)
            assert torch.equal(p1[0], p[i]) and torch.equal(s1[0], s[i])
        p2, s2 = cb.psnr_ssim(_dev(a), _dev(b), 0, y)                 # repeated runs: bit-identical
        assert torch.equal(p, p2) and torch.equal(s, s2)


@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
def test_identical_images(dtype):
    a = pair(dtype, 64, 70, seed=5)[0]
    for y in (False, True):
        assert cb.calculate_psnr(a, a.copy(), 3, test_y_channel=y) == float('inf')
        assert cb.calculate_ssim(a, a.copy(), 3, test_y_channel=y) == 1.0
        p, s = cb.psnr_ssim(_dev(np.stack([a, a])), _dev(np.stack([a, a])), 0, y)
        assert torch.isinf(p).all() and bool((s == 1.0).all())


def test_sweep_form():
    rng = np.random.default_rng(7)
    gt = rng.integers(0, 256, (3, 96, 80, 3), dtype=np.uint8)
    cand = np.clip(gt[:, None].astype(int) + rng.integers(-30, 31, (3, 4, 96, 80, 3)), 0, 255).astype(np.uint8)
    for y in (False, True):
        p, s = cb.psnr_ssim(_dev(cand), _dev(gt), 2, y)
        assert p.shape == s.shape == (3, 4)
        for k in range(4):
            pk, sk = cb.psnr_ssim(_dev(cand[:, k]), _dev(gt), 2, y)
            assert torch.equal(p[:, k], pk) and torch.equal(s[:, k], sk)
        check_psnr(float(p[1, 2]), MO.psnr(cand[1, 2], gt[1], 2, 'HWC', y), np.uint8, y, False)
        assert abs(float(s[1, 2]) - MO.ssim(cand[1, 2], gt[1], 2, 'HWC', y)) <= SSIM_BAR


def test_real_fidelity_sweep():
    """psnr_ssim of a forward_u8_sweep output against its input faces, next to identity_similarity's [B,K]."""
    faces = torch.from_numpy(np.load(os.path.join(GOLDEN, 'faces.npz'))['faces'][:3]).to(DEV)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    sweep = cf.forward_u8_sweep(faces, [0.0, 0.5, 1.0])
    p, s = cb.psnr_ssim(sweep, faces)
    assert p.shape == s.shape == (3, 3)
    for k in range(3):
        pk, sk = cb.psnr_ssim(sweep[:, k].contiguous(), faces)
        assert torch.equal(p[:, k], pk) and torch.equal(s[:, k], sk)
    r, g = sweep[2, 1].cpu().numpy(), faces[2].cpu().numpy()
    assert cb.calculate_psnr(sweep[2, 1], faces[2], 0) == MO.psnr(r, g, 0)
    assert abs(float(p[2, 1]) - MO.psnr(r, g, 0)) <= PSNR_INT_BAR
    assert abs(float(s[2, 1]) - MO.ssim(r, g, 0)) <= SSIM_BAR
    print('sweep psnr', p.cpu().numpy(), 'ssim', s.cpu().numpy())


def test_list_form_on_restored_images(nets):   # noqa: F811
    base = whole_images()
    imgs = [_to_gray(base[1]), base[2], base[-1]]
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser)
    gts = [cv2.resize(im, (r.shape[1], r.shape[0]), interpolation=cv2.INTER_CUBIC) for im, r in zip(imgs, res)]
    # a gray image's 16-bit canvas (a colour transfer that went above 256), against its uint8 ground truth
    img, invs, restored, cropped, _ = _paste_inputs(1)
    faces = cb.gray_adain_faces(torch.from_numpy(restored).to(DEV), torch.from_numpy(cropped).to(DEV))
    faces[1] = faces[1] * 0.2 + 270.0
    wide, _ = PB._paste(torch.from_numpy(img).to(DEV), faces, invs, 1, 512, None, None)
    assert wide.dtype == torch.uint16
    res, gts = list(res) + [wide], gts + [img]
    for y in (False, True):
        p, s = cb.psnr_ssim(res, gts, 4, y)
        assert p.shape == s.shape == (len(res),)
        for i, (r, g) in enumerate(zip(res, gts)):
            dp, ds = cb.calculate_psnr(r, g, 4, test_y_channel=y), cb.calculate_ssim(r, g, 4, test_y_channel=y)
            assert abs(float(p[i]) - dp) <= PSNR_INT_BAR and float(s[i]) == ds
            rn = r.cpu().numpy() if torch.is_tensor(r) else r
            check_psnr(dp, MO.psnr(rn, g, 4, 'HWC', y), np.float64 if rn.dtype != g.dtype else rn.dtype, y, True)
            assert abs(ds - MO.ssim(rn, g, 4, 'HWC', y)) <= SSIM_BAR
        # restore_images_sweep's results[k][i] against one ground truth each: [K, N]
        other = [np.ascontiguousarray(r[::-1]) if isinstance(r, np.ndarray) else r.flip(0).contiguous() for r in res]
        pk, sk = cb.psnr_ssim([res, other], gts, 4, y)
        assert pk.shape == (2, len(res)) and torch.equal(pk[0], p) and torch.equal(sk[0], s)
        q, t = cb.psnr_ssim(other, gts, 4, y)
        assert torch.equal(pk[1], q) and torch.equal(sk[1], t)
    cb.check_async_status()


def test_mixed_dtypes():
    a, b = pair(np.uint8, 50, 60, seed=8)
    for y in (False, True):
        assert cb.calculate_psnr(a, b.astype(np.float64), 2, test_y_channel=y) == \
            cb.calculate_psnr(a.astype(np.float64), b.astype(np.float64), 2, test_y_channel=y)
        assert cb.calculate_ssim(_dev(a), b.astype(np.float32), 2, test_y_channel=y) == cb.calculate_ssim(a, b, 2, test_y_channel=y)


def test_errors_and_nan():
    a, b = pair(np.uint8, 30, 30, seed=9)
    with pytest.raises(AssertionError):
        cb.calculate_psnr(a, b[:, :-1], 0)
    with pytest.raises(ValueError, match='input_order'):
        cb.calculate_ssim(a, b, 0, 'HCW')
    with pytest.raises(ValueError, match='crop_border'):
        cb.calculate_psnr(a, b, -1)
    with pytest.raises(ValueError, match='crop_border'):
        cb.psnr_ssim(_dev(a)[None], _dev(b)[None], -2)
    with pytest.raises(ValueError):
        cb.psnr_ssim(_dev(a)[None], _dev(b)[None], 10)                # 10 x 10 left: under SSIM's 11
    with pytest.raises(NotImplementedError):
        cb.calculate_psnr(a.astype(np.int32), b.astype(np.int32), 0)
    with pytest.raises(NotImplementedError):
        cb.calculate_ssim(_dev(a).half(), _dev(b).half(), 0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.calculate_psnr(torch.from_numpy(a), torch.from_numpy(b), 0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.psnr_ssim(torch.from_numpy(a)[None], torch.from_numpy(b)[None])
    with pytest.raises(ValueError):
        cb.psnr_ssim(_dev(a)[None], _dev(b)[None, :, :-1])
    with pytest.raises(ValueError):
        cb.psnr_ssim([a, a], [b])
    f, g = pair(np.float32, 40, 40, seed=10)
    f[7, 9, 2] = np.nan
    assert np.isnan(cb.calculate_psnr(f, g, 0)) and np.isnan(cb.calculate_ssim(f, g, 0))
    h = g.copy()
    h[3, 3, 0] = np.inf
    p, s = cb.psnr_ssim(_dev(np.stack([f, h, g])), _dev(np.stack([g, g, g])), 0, True)
    torch.cuda.synchronize()
    assert torch.isnan(p[0]) and torch.isnan(s[0]) and torch.isinf(p[2]) and float(s[2]) == 1.0
    assert not torch.isfinite(p[1])
    cb.check_async_status()
