"""not gpu: the colour and mask stages of FFHQBlindDataset.  The sampler's new draws against the UNMODIFIED reference
(brush_stroke_mask, color_jitter_pt and the draw order of __getitem__; skips without the reference tree), the restatement
(oracle/degradation_color_oracle.py) against cv2 and torchvision, and the whole colorization and inpainting inputs against
the unmodified dataset class."""
import importlib.util
import math
import os
import random
import sys
import types

import cv2
import numpy as np
import pytest
import torch

from codeformer_b200 import degradation as DG
from oracle import degradation_color_oracle as CO
from oracle import degradation_oracle as DO
from oracle import ref_shim

F32 = np.float32
TV_RANGES = dict(brightness=(0.5, 1.5), contrast=(0.5, 1.5), saturation=(0, 1.5), hue=(-0.1, 0.1))


def _reference_data():
    """basicsr.data.data_util and basicsr.data.ffhq_blind_dataset, imported unmodified with bare ``basicsr`` and
    ``basicsr.data`` packages (their __init__ chains need modules this environment lacks)."""
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    sys.dont_write_bytecode = True
    for name in ('basicsr', 'basicsr.data'):
        if name not in sys.modules or not hasattr(sys.modules[name], '__path__'):
            m = types.ModuleType(name)
            m.__path__ = [os.path.join(ref_shim.REF_ROOT, *name.split('.'))]
            sys.modules[name] = m
    from basicsr.data import data_util, ffhq_blind_dataset
    return data_util, ffhq_blind_dataset


def _reference_kernels():
    path = os.path.join(ref_shim.REF_ROOT, 'basicsr', 'data', 'gaussian_kernels.py')
    spec = importlib.util.spec_from_file_location('_ref_gaussian_kernels_color', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _Recorder:
    """Stands in for PIL.ImageDraw in data_util: forwards every call to the real ImageDraw and records the geometry."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def Draw(self, img):                   # noqa: N802 (PIL's name)
        draw, calls = self.real.Draw(img), self.calls

        class D:
            def line(self, xy, **kw):
                calls.append(('line', list(xy), kw['width']))
                draw.line(xy, **kw)

            def ellipse(self, xy, **kw):
                calls.append(('ellipse', tuple(xy)))
                draw.ellipse(xy, **kw)
        return D()


def _stroke_calls(strokes):
    out = []
    for vertices, w in strokes:
        out.append(('line', list(vertices), w))
        out += [('ellipse', (x - w // 2, y - w // 2, x + w // 2, y + w // 2)) for x, y in vertices]
    return out

# ------------------------------------------------------------------------------------------------ sampler vs reference


def _replay_reference(du, fb, gk, task, S=512):
    """The draws of ffhq_blind_dataset.py:203-273 for one face, in its order, with the reference's own functions where
    they exist (random_mixed_kernels, brush_stroke_mask, color_jitter_pt with its adjust_* recorded)."""
    out = {}
    if task == 'colorization':
        r = DG.STAGE2_RANGES
        gk.random_mixed_kernels(['iso', 'aniso'], [0.5, 0.5], 41, r['blur_sigma'], r['blur_sigma'], [-math.pi, math.pi],
                                noise_range=None)
        scale = np.random.uniform(*r['downsample_range'])
        size = int(S // scale)
        np.random.uniform(r['noise_range'][0] / 255., r['noise_range'][1] / 255.)
        np.random.randn(size, size, 3)
        np.random.uniform(*r['jpeg_range'])
        if np.random.uniform() < 0.3:
            out['jitter'] = np.random.uniform(-20 / 255., 20 / 255., 3).astype(np.float32)
        out['gray'] = bool(np.random.uniform() < 0.01)
        if np.random.uniform() < 0.3:
            rec = []
            saved = {k: getattr(fb, k) for k in ('adjust_brightness', 'adjust_contrast', 'adjust_saturation', 'adjust_hue')}
            try:
                for k in saved:
                    setattr(fb, k, lambda img, f, _k=k: (rec.append((_k[len('adjust_'):], f)), img)[1])
                fb.FFHQBlindDataset.color_jitter_pt(torch.zeros(3, 1, 1), TV_RANGES['brightness'], TV_RANGES['contrast'],
                                                    TV_RANGES['saturation'], TV_RANGES['hue'])
            finally:
                for k, v in saved.items():
                    setattr(fb, k, v)
            out['jitter_pt'] = rec
    else:
        from PIL import Image
        rec = _Recorder(du.ImageDraw)
        du.ImageDraw = rec
        try:
            img = du.brush_stroke_mask(Image.fromarray(np.zeros((S, S, 3), np.uint8)))
        finally:
            du.ImageDraw = rec.real
        out['mask'] = np.array(img)
        out['calls'] = rec.calls
    return out


@pytest.mark.parametrize('task', ['colorization', 'inpainting'])
def test_sampler_matches_reference_draws(task):
    du, fb = _reference_data()
    gk = _reference_kernels()
    opts = DG.COLORIZATION_OPTIONS if task == 'colorization' else DG.INPAINTING_OPTIONS
    seen = {'jitter': 0, 'gray': 0, 'jitter_pt': 0}
    for seed in range(200):
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        ref = _replay_reference(du, fb, gk, task)
        state = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state())
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        p = DG.sample_degradations(1, **opts)[0]
        assert random.getstate() == state[0]
        assert np.array_equal(np.random.get_state()[1], state[1]), (seed, 'np.random consumed differently')
        assert torch.equal(torch.get_rng_state(), state[2]), (seed, 'the torch generator consumed differently')
        if task == 'colorization':
            assert (p['jitter'] is None) == ('jitter' not in ref)
            if p['jitter'] is not None:
                assert p['jitter'].dtype == np.float32 and np.array_equal(p['jitter'], ref['jitter'])
            assert p['gray'] == ref['gray']
            assert (p['jitter_pt'] or []) == ref.get('jitter_pt', [])
            assert p['mask'] is None and p['strokes'] is None
            seen['jitter'] += p['jitter'] is not None
            seen['gray'] += p['gray']
            seen['jitter_pt'] += p['jitter_pt'] is not None
        else:
            assert p['kernel'] is None and p['size'] is None and p['jitter'] is None and not p['gray']
            assert _stroke_calls(p['strokes']) == ref['calls'], seed
            assert np.array_equal(p['mask'], ref['mask'][..., 0]) and (ref['mask'] == ref['mask'][..., :1]).all(), seed
    if task == 'colorization':
        assert seen['jitter'] > 30 and seen['jitter_pt'] > 30 and seen['gray'] >= 1, seen


def test_sampler_defaults_unchanged_and_options():
    rs_a, rs_b = np.random.RandomState(1), np.random.RandomState(1)
    a = DG.sample_degradations(3, py_rng=random.Random(1), np_rng=rs_a)
    b = DG.sample_degradations(3, py_rng=random.Random(1), np_rng=rs_b, color_jitter_prob=None, gray_prob=0.0,
                               color_jitter_pt_prob=None, gen_inpaint_mask=False, torch_rng=torch.Generator())
    assert np.array_equal(rs_a.get_state()[1], rs_b.get_state()[1]) and rs_a.get_state()[2] == rs_b.get_state()[2]
    for x, y in zip(a, b):
        assert x['size'] == y['size'] and np.array_equal(x['kernel'], y['kernel']) and np.array_equal(x['noise'], y['noise'])
        assert (x['jitter'], x['gray'], x['jitter_pt'], x['strokes'], x['mask']) == (None, False, None, None, None)
    g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    before = torch.get_rng_state()
    p = DG.sample_degradations(20, np_rng=np.random.RandomState(2), color_jitter_pt_prob=1.0, torch_rng=g1, hue=None)
    assert torch.equal(before, torch.get_rng_state()), 'an explicit generator leaves the default one alone'
    q = DG.sample_degradations(20, np_rng=np.random.RandomState(2), color_jitter_pt_prob=1.0, torch_rng=g2, hue=None)
    assert [x['jitter_pt'] for x in p] == [x['jitter_pt'] for x in q]
    assert all(len(x['jitter_pt']) == 3 and 'hue' not in dict(x['jitter_pt']) for x in p)
    with pytest.raises(ValueError):
        DG.sample_degradations(1, gt_size=512, in_size=256, use_corrupt=False)
    m = DG.sample_degradations(2, gt_size=128, in_size=128, np_rng=np.random.RandomState(0), **DG.INPAINTING_OPTIONS)
    assert all(x['mask'].shape == (128, 128) and x['mask'].dtype == np.uint8 and x['mask'].max() == 255 for x in m)

# ---------------------------------------------------------------------------------------------- oracle vs cv2 / tv


def _tvf():
    return pytest.importorskip('torchvision.transforms.functional')


def _faces(n=3, h=48, w=40, seed=0):
    """Random, smooth and special-content float32 RGB [3, h, w] images: gray pixels (s = 0), pure and saturated colours,
    black and white, and hues on both sides of red (the wrap-around)."""
    rng = np.random.default_rng(seed)
    out = [torch.from_numpy(rng.random((3, h, w), dtype=np.float32)) for _ in range(n)]
    smooth = cv2.GaussianBlur(rng.random((h, w, 3), dtype=np.float32), (9, 9), 3).transpose(2, 0, 1)
    out.append(torch.from_numpy(np.ascontiguousarray(smooth)))
    special = rng.random((3, h, w), dtype=np.float32)
    k = (rng.integers(0, 256, (h, w)).astype(np.float32) / F32(255.))
    special[:, : h // 4] = k[None, : h // 4]                                 # gray
    pure = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1], [1, 1, 1], [0, 0, 0]], np.float32)
    special[:, h // 4: h // 2] = pure[rng.integers(0, 8, (h // 4, w))].transpose(2, 0, 1)
    wrap = np.stack([np.ones((h // 4, w), np.float32), rng.random((h // 4, w), dtype=np.float32) * 0.05,
                     rng.random((h // 4, w), dtype=np.float32) * 0.05])          # red with a little g or b: h near 0 / 1
    special[:, h // 2: 3 * h // 4] = wrap[[0, 1, 2]] if seed % 2 == 0 else wrap[[0, 2, 1]]
    out.append(torch.from_numpy(special))
    return out


def test_gray_bit_equal_to_cv2():
    rng = np.random.default_rng(1)
    for shape in [(1, 1), (3, 5), (31, 33), (512, 512), (100, 37)]:
        x = rng.random(shape + (3,), dtype=np.float32)
        assert np.array_equal(CO.gray_cv2(x), cv2.cvtColor(x, cv2.COLOR_BGR2GRAY)), shape
    x = (rng.integers(0, 256, (64, 64, 3)).astype(np.float32) / F32(255.)).astype(np.float32)
    assert np.array_equal(CO.gray_cv2(x), cv2.cvtColor(x, cv2.COLOR_BGR2GRAY))


OP_FACTORS = {'brightness': [0.5, 0.73, 1.0, 1.3, 1.5], 'contrast': [0.5, 0.81, 1.0, 1.5],
              'saturation': [0.0, 0.4, 1.0, 1.5], 'hue': [-0.1, -0.04, 0.0, 0.06, 0.1, -0.5, 0.5]}


@pytest.mark.parametrize('op', list(OP_FACTORS))
def test_each_op_bit_equal_to_torchvision(op):
    F = _tvf()
    fn = getattr(F, f'adjust_{op}')
    for seed in range(2):
        for img in _faces(seed=seed):
            for f in OP_FACTORS[op]:
                f = float(np.float32(f))
                got, _ = CO.apply_ops(img, [(op, f)])
                assert torch.equal(got, fn(img, f)), (op, f)
    if op == 'contrast':
        img = _faces()[0]
        m = float(CO.contrast_mean(img))
        assert torch.equal(CO.adjust_contrast(img, 0.7, m), F.adjust_contrast(img, 0.7))


def test_color_jitter_pt_all_24_orders():
    """The reference's color_jitter_pt and the oracle fed the sampler's draws of the same torch seed, until every one of
    the 24 orders has come up."""
    _, fb = _reference_data()
    img = _faces(1, 24, 20)[-1]
    orders = set()
    for seed in range(2000):
        torch.manual_seed(seed)
        want = fb.FFHQBlindDataset.color_jitter_pt(img, *TV_RANGES.values())
        torch.manual_seed(seed)
        ops = DG._draw_jitter_pt(tuple(TV_RANGES.values()), None)
        got, _ = CO.apply_ops(img, ops)
        assert torch.equal(got, want), (seed, ops)
        orders.add(tuple(op for op, _ in ops))
        if len(orders) == 24:
            break
    assert len(orders) == 24


def test_uint8_round_trip_without_corruption():
    """float32(k / 255) * 255 rounds back to k, and so does the mask path's float32(float64(k / 255)) * 255 truncated or
    rounded: a face without stages is gt, and a masked face is where(mask, 255, gt)."""
    k = np.arange(256)
    a = (k.astype(F32) / F32(255.)).astype(F32)
    b = (k / 255.).astype(F32)
    assert np.array_equal(CO.round_u8(a), k) and np.array_equal((a * F32(255.)).astype(np.uint8), k)
    assert np.array_equal(CO.round_u8(b), k)

# ------------------------------------------------------------------------------------------- the unmodified dataset


def _run_dataset(fb, folder, opt_extra, seed, patch_blur=True):
    """FFHQBlindDataset.__getitem__(0) with mean 0, std 1, no flips; returns (uint8 BGR input, recorded contrast means).
    With patch_blur the dataset's cv2.filter2D is replaced by the float64 direct sum (the reference's filter2D uses a DFT for
    41 x 41 kernels), so the chain starts from the same blurred image as the oracle; everything else is the class's own."""
    opt = dict(dataroot_gt=folder, io_backend={'type': 'disk'}, use_hflip=False, mean=[0., 0., 0.], std=[1., 1., 1.],
               gt_size=64, in_size=64, **opt_extra)
    ds = fb.FFHQBlindDataset(opt)
    means = []
    real_cv2, real_contrast = fb.cv2, fb.adjust_contrast

    class Cv2:
        def __getattr__(self, name):
            return getattr(real_cv2, name)

        @staticmethod
        def filter2D(img, ddepth, kernel):        # noqa: N802 (cv2's name)
            return DO.filter2d_f64(img, kernel)

    def contrast(img, f):
        means.append(float(CO.contrast_mean(img)))
        return real_contrast(img, f)
    fb.adjust_contrast = contrast
    if patch_blur:
        fb.cv2 = Cv2()
    try:
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        out = ds[0]['in']
    finally:
        fb.cv2, fb.adjust_contrast = real_cv2, real_contrast
    rgb = (out * 255.).round().clamp(0, 255).to(torch.uint8).numpy().transpose(1, 2, 0)
    return np.ascontiguousarray(rgb[..., ::-1]), means


def _write_face(tmp_path):
    rng = np.random.default_rng(3)
    face = cv2.GaussianBlur(rng.integers(0, 256, (64, 64, 3)).astype(np.uint8), (7, 7), 2)
    cv2.imwrite(str(tmp_path / 'face.png'), face)
    return face


def test_inpainting_inputs_equal_the_dataset(tmp_path):
    _, fb = _reference_data()
    face = _write_face(tmp_path)
    for seed in range(12):
        want, _ = _run_dataset(fb, str(tmp_path), dict(use_corrupt=False, gen_inpaint_mask=True), seed, patch_blur=False)
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        p = DG.sample_degradations(1, gt_size=64, in_size=64, **DG.INPAINTING_OPTIONS)[0]
        got, _ = CO.degrade_color(face, p, 64)
        assert np.array_equal(got, want), (seed, int((got != want).sum()))


def test_colorization_inputs_equal_the_dataset(tmp_path):
    _, fb = _reference_data()
    face = _write_face(tmp_path)
    opts = dict(COLOR_DATASET, color_jitter_prob=1.0, color_jitter_pt_prob=1.0)
    seen_gray = False
    for seed in range(24):
        gray = seed % 6 == 5
        o = dict(opts, gray_prob=1.0 if gray else 0.0)
        want, means = _run_dataset(fb, str(tmp_path), o, seed)
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        p = DG.sample_degradations(1, gt_size=64, in_size=64, **o)[0]
        assert p['gray'] == gray and p['jitter'] is not None and p['jitter_pt'] is not None
        seen_gray |= p['gray']
        got, used = CO.degrade_color(face, p, 64, means[0] if means else None)
        assert (used is None) == (not means)
        assert np.array_equal(got, want), (seed, int((got != want).sum()))
    assert seen_gray


COLOR_DATASET = dict(use_corrupt=True, blur_kernel_size=41, kernel_list=['iso', 'aniso'], kernel_prob=[0.5, 0.5],
                     blur_sigma=[1, 15], downsample_range=[4, 30], noise_range=[0, 20], jpeg_range=[30, 80],
                     color_jitter_shift=20)
