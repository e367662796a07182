"""-m gpu: synthetic degradations on the device (codeformer_b200.degradation, cfb_degrade_faces / cfb_jpeg_roundtrip) against
cv2 and the numpy restatement (oracle/degradation_oracle.py): the JPEG stage byte for byte, the blurred and downsampled
image within float32 ulps, the later stages byte for byte from the device's own downsampled image, the whole chain against
the host chain, batching, determinism and the errors."""
import ctypes
import random

import cv2
import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import degradation as DG
from oracle import degradation_oracle as DO
from tests.test_oracle_degradation import (JPEG_QUALITIES, JPEG_SIZES, cv2_jpeg, host_chain, jpeg_contents)
from tests.util import golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def gt_faces(n, size=512):
    """n uint8 BGR faces: the committed ones, mirrored and shifted to make more."""
    f = golden('faces.npz')['faces'][..., ::-1]
    out = []
    for i in range(n):
        x = f[i % 4]
        if (i // 4) % 2:
            x = x[:, ::-1]
        x = np.roll(x, 7 * (i // 8), axis=0)
        if size != 512:
            x = cv2.resize(np.ascontiguousarray(x), (size, size), interpolation=cv2.INTER_AREA)
        out.append(np.ascontiguousarray(x))
    return np.stack(out)


def params_for(n, seed, gt_size=512, in_size=512, **ranges):
    return DG.sample_degradations(n, gt_size=gt_size, in_size=in_size, py_rng=random.Random(seed),
                                  np_rng=np.random.RandomState(seed), **ranges)


def run_debug(gt, params, in_size):
    lq, a, pre = DG._run(torch.from_numpy(gt).to(DEV), params, in_size, debug=True)
    torch.cuda.synchronize()
    a, pre = a.cpu().numpy(), pre.cpu().numpy()
    out_a, out_pre, at = [], [], 0
    for p in params:
        n = p['size'] ** 2 * 3
        out_a.append(a[at:at + n].reshape(p['size'], p['size'], 3))
        out_pre.append(pre[at:at + n].reshape(p['size'], p['size'], 3))
        at += n
    return lq.cpu().numpy(), out_a, out_pre


def ulps(got, want):
    sp = np.spacing(np.maximum(np.abs(got), np.abs(want)).astype(np.float32)).astype(np.float64)
    return (np.abs(got.astype(np.float64) - want.astype(np.float64)) / sp).max()

# ---------------------------------------------------------------------------------------------------------------- JPEG


@pytest.mark.parametrize('size', JPEG_SIZES, ids=lambda s: f'{s[0]}x{s[1]}')
def test_jpeg_roundtrip_matches_cv2(size):
    imgs, qs = [], []
    for img in jpeg_contents(*size).values():
        for q in JPEG_QUALITIES:
            imgs.append(img)
            qs.append(q)
    got = cb.jpeg_roundtrip(np.stack(imgs), qs).cpu().numpy()          # mixed qualities in one batch
    for g, img, q in zip(got, imgs, qs):
        assert np.array_equal(g, cv2_jpeg(img, q)), (size, q)
    one = cb.jpeg_roundtrip(torch.from_numpy(imgs[3][None]).to(DEV), qs[3]).cpu().numpy()[0]
    assert np.array_equal(one, got[3])


def test_jpeg_every_quality_in_one_batch():
    img = gt_faces(1, 512)[0, 100:164, 200:280]
    got = cb.jpeg_roundtrip(np.repeat(img[None], 100, 0), list(range(1, 101))).cpu().numpy()
    for q in range(1, 101):
        assert np.array_equal(got[q - 1], cv2_jpeg(img, q)), q

# ------------------------------------------------------------------------------------------------------------ stages


def _check_stages(gt, params, in_size, exact_oracle_faces=2):
    lq, stage_a, pre = run_debug(gt, params, in_size)
    for i, p in enumerate(params):
        # stage a: bit-equal to the restatement, which sums the blur in the device's order.  cv2 filters a 41 x 41 kernel
        # by DFT, whose error is absolute (about 3e-8 on [0, 1] images; up to 2^-23 after the two lerps over the committed
        # faces), so near black it spans several ulps of the value: that bar is two ulps of 1.0.
        if i < exact_oracle_faces:
            _, want_a, _ = DO.degrade(gt[i], p, in_size)
            assert np.array_equal(stage_a[i], want_a), (i, p['size'], ulps(stage_a[i], want_a))
        img = cv2.filter2D(gt[i].astype(np.float32) / 255., -1, p['kernel'])
        cv_a = cv2.resize(img, (p['size'], p['size']), interpolation=cv2.INTER_LINEAR)
        assert np.abs(stage_a[i].astype(np.float64) - cv_a).max() <= 2 * 2. ** -23, (i, p['size'])
        # stages b-d byte-exact from the device's own stage-a image
        x = stage_a[i]
        if p['noise'] is not None:
            x = np.clip(x + p['noise'], 0, 1)
        if p['quality'] is not None:
            assert np.array_equal(pre[i], DO.to_u8(x * np.float32(255.)))
            _, enc = cv2.imencode('.jpg', x * 255., [int(cv2.IMWRITE_JPEG_QUALITY), p['quality']])
            x = np.float32(cv2.imdecode(enc, 1)) / 255.
        x = cv2.resize(x, (in_size, in_size), interpolation=cv2.INTER_LINEAR)
        want = np.clip((x * 255.).round(), 0, 255).astype(np.uint8)
        assert np.array_equal(lq[i], want), (i, p['size'], p['quality'], int((lq[i] != want).sum()))
    return lq, stage_a, pre


@pytest.mark.parametrize('stage', ['stage2', 'stage3'])
def test_stages_exact_batch32(stage):
    r = DG.STAGE2_RANGES if stage == 'stage2' else DG.STAGE3_RANGES
    gt = gt_faces(32)
    params = params_for(32, 11, **r)
    _check_stages(gt, params, 512)


@pytest.mark.parametrize('stage', ['stage2', 'stage3'])
def test_stage_a_bit_equal_to_restatement(stage):
    """Every face of a batch at gt_size 128: small sizes 4 .. 128, sampled and full blur grids."""
    r = DG.STAGE2_RANGES if stage == 'stage2' else DG.STAGE3_RANGES
    gt = gt_faces(12, 128)
    params = params_for(12, 17, gt_size=128, in_size=128, **r)
    _check_stages(gt, params, 128, exact_oracle_faces=12)


def test_stages_without_noise_or_jpeg():
    gt = gt_faces(4)
    for kw in (dict(noise_range=None), dict(jpeg_range=None), dict(noise_range=None, jpeg_range=None)):
        params = params_for(4, 3, **dict(DG.STAGE2_RANGES, **kw))
        _check_stages(gt, params, 512, exact_oracle_faces=0)


def test_gt256_and_smaller_in_size():
    gt = gt_faces(3, 256)
    params = params_for(3, 8, gt_size=256, in_size=128, blur_sigma=(1, 15), downsample_range=(1, 12), noise_range=(0, 20),
                        jpeg_range=(30, 80))
    _check_stages(gt, params, 128, exact_oracle_faces=1)
    lq, _ = cb.degrade_faces(gt, params, in_size=128)
    assert lq.shape == (3, 128, 128, 3) and lq.dtype == torch.uint8

# ------------------------------------------------------------------------------------------------------- whole chain


def test_whole_chain_against_host_chain():
    """From the same GT and parameters: a byte differs from the host chain only where the JPEG input (or, without JPEG, the
    float image) differed -- the blur's last-ulp differences -- and those inputs differ by at most 1."""
    gt = gt_faces(8)
    params = params_for(8, 21, **DG.STAGE2_RANGES)
    lq, stage_a, pre = run_debug(gt, params, 512)
    equal = total = 0
    for i, p in enumerate(params):
        want = host_chain(gt[i], p, 512)
        equal += int((lq[i] == want).sum())
        total += want.size
        img = cv2.filter2D(gt[i].astype(np.float32) / 255., -1, p['kernel'])
        x = np.clip(cv2.resize(img, (p['size'], p['size']), interpolation=cv2.INTER_LINEAR) + p['noise'], 0, 1)
        host_pre = DO.to_u8(x * np.float32(255.))
        d = np.abs(pre[i].astype(int) - host_pre)
        assert d.max() <= 1
        # MCUs whose input differed, grown by one MCU (the decoder's chroma upsampling reads the neighbours)
        s = p['size']
        m = -(-s // 16)
        dirty = np.zeros((m + 2, m + 2), bool)
        ys, xs = np.nonzero(d.max(2))
        dirty[ys // 16 + 1, xs // 16 + 1] = True
        dirty = dirty | np.roll(dirty, 1, 0) | np.roll(dirty, -1, 0)
        dirty = dirty | np.roll(dirty, 1, 1) | np.roll(dirty, -1, 1)
        y0, y1, _ = DO.linear_taps(512, s)
        oy, ox = np.nonzero((lq[i] != want).any(2))
        ok = dirty[y0[oy] // 16 + 1, y0[ox] // 16 + 1] | dirty[y1[oy] // 16 + 1, y1[ox] // 16 + 1] | \
            dirty[y0[oy] // 16 + 1, y1[ox] // 16 + 1] | dirty[y1[oy] // 16 + 1, y0[ox] // 16 + 1]
        assert ok.all(), (i, int((~ok).sum()))
    print(f'whole chain: {equal / total:.6f} of the bytes equal the host chain')
    assert equal / total > 0.9

# --------------------------------------------------------------------------------------------------- batches, errors


def test_batches_equal_per_face_calls_and_repeat():
    gt = gt_faces(32)
    params = params_for(32, 5, **DG.STAGE3_RANGES)
    assert len({p['size'] for p in params}) > 10
    full, _ = cb.degrade_faces(gt, params)
    again, _ = cb.degrade_faces(torch.from_numpy(gt).to(DEV), params)
    assert torch.equal(full, again)
    three, _ = cb.degrade_faces(gt[5:8], params[5:8])
    assert torch.equal(three, full[5:8])
    for i in (0, 17, 31):
        one, _ = cb.degrade_faces(gt[i:i + 1], params[i:i + 1])
        assert torch.equal(one[0], full[i])


def test_default_sampling_uses_global_rngs():
    gt = gt_faces(2)
    random.seed(4)
    np.random.seed(4)
    lq, params = cb.degrade_faces(gt)
    random.seed(4)
    np.random.seed(4)
    want = DG.sample_degradations(2)
    assert [p['size'] for p in params] == [p['size'] for p in want]
    assert torch.equal(lq, cb.degrade_faces(gt, want)[0])


def test_errors():
    gt = gt_faces(1)
    p = params_for(1, 0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.degrade_faces(torch.from_numpy(gt), p)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.jpeg_roundtrip(torch.from_numpy(gt), 50)
    with pytest.raises(NotImplementedError):
        cb.degrade_faces(gt.astype(np.float32), p)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt[:, :, :500], p)
    with pytest.raises(ValueError):
        cb.degrade_faces(np.zeros((1, 64, 64, 4), np.uint8), p)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, p, in_size=1024)
    bad = [dict(p[0], quality=101)]
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, bad)
    with pytest.raises(ValueError):
        cb.jpeg_roundtrip(gt, 0)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, p + p)
    lib = cb._lib.load()
    assert lib.cfb_degrade_workspace_bytes(1, 512, (ctypes.c_int32 * 1)(600), None) == -1
