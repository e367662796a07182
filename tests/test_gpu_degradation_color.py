"""-m gpu: the colour and mask stages on the device (codeformer_b200.degradation, cfb_degrade_faces_color) against the
restatement (oracle/degradation_color_oracle.py) given the device's contrast means: each op alone, all 24 orders, the shift
with clipping, gray, masks, the colorization chain at B = 32 and mixed batches; the contrast mean against the exact mean and
torch's; faces without the new stages against the chain's own path; batching, determinism and the errors."""
import itertools
import math
import random

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import degradation as DG
from oracle import degradation_color_oracle as CO
from tests.test_gpu_degradation import gt_faces, params_for

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F32 = np.float32
RANGES = {'brightness': (0.5, 1.5), 'contrast': (0.5, 1.5), 'saturation': (0, 1.5), 'hue': (-0.1, 0.1)}


def f32(x):
    return float(np.float32(x))


def run_color(gt, params, in_size):
    lq, means = DG._run_color(torch.from_numpy(gt).to(DEV), params, in_size, debug=True)
    return lq.cpu().numpy(), means.cpu().numpy()


def stage_a(gt, params, in_size):
    """The device's downsampled image of each corrupted face, from the chain's own debug path."""
    _, a, _ = DG._run(torch.from_numpy(gt).to(DEV), params, in_size, debug=True)
    a, out, at = a.cpu().numpy(), [], 0
    for p in params:
        n = p['size'] ** 2 * 3
        out.append(a[at:at + n].reshape(p['size'], p['size'], 3))
        at += n
    return out


def oracle(gt, params, in_size, means):
    """Per face the restatement from the device's stage-a image (cv2's DFT blur is not what either side runs), with the
    device's contrast mean."""
    corrupt = params[0]['kernel'] is not None
    a = stage_a(gt, params, in_size) if corrupt else None
    out = []
    for i, p in enumerate(params):
        if p.get('mask') is not None:
            out.append(CO.degrade_color(gt[i], p, in_size)[0])
            continue
        x = CO.finish_chain(a[i], p, in_size) if corrupt else CO.chain_float(gt[i], p, in_size)
        has_contrast = any(op == 'contrast' for op, _ in (p.get('jitter_pt') or []))
        got, _ = CO.color_stages(x, p, means[i] if has_contrast else None)
        out.append(got)
    return np.stack(out)


def check(gt, params, in_size):
    lq, means = run_color(gt, params, in_size)
    want = oracle(gt, params, in_size, means)
    for i in range(len(params)):
        assert np.array_equal(lq[i], want[i]), (i, params[i].get('jitter_pt'), int((lq[i] != want[i]).sum()))
    return lq, means


def with_stages(params, **kw):
    return [dict(p, **{k: (v[i] if isinstance(v, list) else v) for k, v in kw.items()}) for i, p in enumerate(params)]

# ------------------------------------------------------------------------------------------------------------- ops


@pytest.mark.parametrize('op', list(RANGES))
def test_each_op_alone(op):
    lo, hi = RANGES[op]
    factors = [lo, hi, (lo + hi) / 2, lo + 0.3 * (hi - lo), 1.0 if op != 'hue' else 0.0, -0.5 if op == 'hue' else 0.0,
               0.5 if op == 'hue' else 2.5, lo + 0.77 * (hi - lo)]
    gt = gt_faces(len(factors), 128)
    params = params_for(len(factors), 3, gt_size=128, in_size=128, **DG.STAGE2_RANGES)
    check(gt, with_stages(params, jitter_pt=[[(op, f32(f))] for f in factors]), 128)


def test_all_24_orders():
    rng = np.random.default_rng(0)
    orders = list(itertools.permutations(RANGES))
    gt = gt_faces(24, 128)
    params = params_for(24, 9, gt_size=128, in_size=128, **DG.STAGE3_RANGES)
    seq = [[(op, f32(rng.uniform(*RANGES[op]))) for op in order] for order in orders]
    check(gt, with_stages(params, jitter_pt=seq), 128)
    # without corruption, and with the shift and gray in front
    seq2 = [[(op, f32(rng.uniform(*RANGES[op]))) for op in order[:2 + i % 3]] for i, order in enumerate(orders)]
    jit = [rng.uniform(-20 / 255., 20 / 255., 3).astype(F32) for _ in orders]
    bare = DG.sample_degradations(24, gt_size=128, in_size=128, use_corrupt=False)
    check(gt, with_stages(bare, jitter_pt=seq2, jitter=jit, gray=[i % 5 == 0 for i in range(24)]), 128)


def test_shift_with_clipping_and_gray():
    rng = np.random.default_rng(1)
    gt = gt_faces(8, 128)
    params = params_for(8, 4, gt_size=128, in_size=128, **DG.STAGE2_RANGES)
    jit = [rng.uniform(-s, s, 3).astype(F32) for s in (20 / 255., 20 / 255., 0.3, 0.3, 0.6, 0.6, 1.0, 1.0)]
    lq, _ = check(gt, with_stages(params, jitter=jit), 128)
    lq_g, _ = check(gt, with_stages(params, jitter=jit, gray=True), 128)
    assert (lq_g[..., 0] == lq_g[..., 1]).all() and (lq_g[..., 1] == lq_g[..., 2]).all()
    check(gt, with_stages(params, gray=True), 128)


def test_masks():
    rng = np.random.default_rng(2)
    gt = gt_faces(6, 256)
    params = DG.sample_degradations(6, gt_size=256, in_size=256, use_corrupt=False)
    yy, xx = np.mgrid[0:256, 0:256]
    masks = []
    for i in range(6):
        m = np.zeros((256, 256), np.uint8)
        for _ in range(3):
            cy, cx, r = rng.integers(0, 256, 2).tolist() + [int(rng.integers(10, 60))]
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 255
        m[rng.integers(0, 256):, :rng.integers(1, 40)] = 1 + i         # any nonzero value masks
        masks.append(m if i != 3 else None)                            # one face without a mask in the batch
    lq, _ = check(gt, with_stages(params, mask=masks), 256)
    for i, m in enumerate(masks):
        want = gt[i] if m is None else np.where(m[..., None] != 0, 255, gt[i])
        assert np.array_equal(lq[i], want)
    # the inpainting preset end to end (PIL-rasterised strokes)
    pytest.importorskip('PIL')
    p = DG.sample_degradations(4, gt_size=256, in_size=256, np_rng=np.random.RandomState(7), **DG.INPAINTING_OPTIONS)
    lq, _ = cb.degrade_faces(gt[:4], p, in_size=256)
    for i in range(4):
        assert np.array_equal(lq[i].cpu().numpy(), np.where(p[i]['mask'][..., None] != 0, 255, gt[i]))

# ------------------------------------------------------------------------------------------------ chains and batches


def colorization_params(n, seed, **over):
    opts = dict(DG.COLORIZATION_OPTIONS, **over)
    return DG.sample_degradations(n, py_rng=random.Random(seed), np_rng=np.random.RandomState(seed),
                                  torch_rng=torch.Generator().manual_seed(seed), **opts)


def test_colorization_chain_batch32():
    gt = gt_faces(32)
    params = colorization_params(32, 11, color_jitter_prob=0.6, color_jitter_pt_prob=0.8, gray_prob=0.2)
    assert sum(p['jitter_pt'] is not None for p in params) > 15 and any(p['gray'] for p in params)
    check(gt, params, 512)
    check(gt, colorization_params(32, 12), 512)         # the preset's own probabilities: most faces without stages


def test_faces_without_stages_equal_the_chain_path():
    gt = gt_faces(12)
    params = colorization_params(12, 5, color_jitter_prob=0.5, color_jitter_pt_prob=0.5)
    lq, _ = check(gt, params, 512)
    plain = [{k: p[k] for k in ('kernel_type', 'sigma_x', 'sigma_y', 'rotation', 'kernel', 'scale', 'size', 'noise_sigma',
                                'noise', 'quality')} for p in params]
    base, _, _ = DG._run(torch.from_numpy(gt).to(DEV), plain, 512, debug=False)
    base = base.cpu().numpy()
    bare = [i for i, p in enumerate(params) if not DG._has_color_stage(p)]
    assert 0 < len(bare) < 12
    for i in bare:
        assert np.array_equal(lq[i], base[i]), i
    # and faces without corruption or stages are the ground truth
    none = DG.sample_degradations(3, gt_size=512, in_size=512, use_corrupt=False)
    assert np.array_equal(cb.degrade_faces(gt[:3], none)[0].cpu().numpy(), gt[:3])


def contrast_state(gt_i, p, in_size, a_i):
    """The float32 RGB image the contrast op sees (restatement, from the device's stage-a image)."""
    x = CO.finish_chain(a_i, p, in_size)
    if p.get('jitter') is not None:
        x = np.clip(x + p['jitter'], 0, 1).astype(F32)
    if p.get('gray'):
        x = np.repeat(CO.gray_cv2(x)[..., None], 3, 2)
    img = torch.from_numpy(np.ascontiguousarray(x[..., ::-1].transpose(2, 0, 1)))
    ops = p['jitter_pt']
    k = [op for op, _ in ops].index('contrast')
    img, _ = CO.apply_ops(img, ops[:k])
    return img


def test_contrast_mean_bounds():
    """The device mean against the exact mean of the same gray values (math.fsum) and against torch's CPU mean.

    Device: float64 block sums of N <= 2^18 float32 values in [0, 1] carry a relative error below N 2^-53 < 3e-11, then
    one rounding to float32: within one float32 ulp of the exact mean (half an ulp but for that float64 error).
    torch: a float32 cascade sum of nonnegative terms; each term passes through at most 4 levels of at most 16 additions,
    then the combination of vector lanes, accumulators and thread chunks (at most log2 N more), so the depth D <= 64 +
    log2 N and the sum's relative error is at most D u / (1 - D u), u = 2^-24; the division adds one u.  Hence
    |device - torch| <= ulp + (D + 2) u mean (1 + 1e-3)."""
    gt = gt_faces(8)
    params = params_for(8, 13, **DG.STAGE2_RANGES)
    rng = np.random.default_rng(3)
    seq = []
    for i in range(8):
        order = list(RANGES)
        rng.shuffle(order)
        seq.append([(op, f32(rng.uniform(*RANGES[op]))) for op in order])
    params = with_stages(params, jitter_pt=seq, gray=[i == 2 for i in range(8)])
    lq, means = check(gt, params, 512)
    a = stage_a(gt, params, 512)
    n = 512 * 512
    D = 64 + math.log2(n)
    u = 2. ** -24
    for i, p in enumerate(params):
        img = contrast_state(gt[i], p, 512, a[i])
        g = CO.rgb_to_gray(img).numpy().astype(np.float64).ravel()
        exact = math.fsum(g) / n
        dev = float(means[i])
        assert abs(dev - exact) <= np.spacing(F32(exact)), (i, dev, exact)
        tmean = float(CO.contrast_mean(img))
        assert abs(dev - tmean) <= np.spacing(F32(exact)) + (D + 2) * u * exact * (1 + 1e-3), (i, dev, tmean)
    no = with_stages(params_for(2, 1, **DG.STAGE2_RANGES), jitter_pt=[[('hue', f32(0.05))], None])
    _, m = run_color(gt[:2], no, 512)
    assert np.isnan(m[:2]).all()


def test_batches_equal_per_face_calls_and_repeat():
    gt = gt_faces(16)
    params = colorization_params(16, 21, color_jitter_prob=0.7, color_jitter_pt_prob=0.9, gray_prob=0.1)
    full, _ = cb.degrade_faces(gt, params)
    again, _ = cb.degrade_faces(torch.from_numpy(gt).to(DEV), params)
    assert torch.equal(full, again)
    for i in (0, 7, 15):
        one, _ = cb.degrade_faces(gt[i:i + 1], params[i:i + 1])
        assert torch.equal(one[0], full[i])
    three, _ = cb.degrade_faces(gt[4:7], params[4:7])
    assert torch.equal(three, full[4:7])


def test_errors():
    gt = gt_faces(2, 128)
    bare = DG.sample_degradations(2, gt_size=128, in_size=128, use_corrupt=False)
    chain = params_for(2, 0, gt_size=128, in_size=128)
    m = np.zeros((128, 128), np.uint8)
    with pytest.raises(NotImplementedError):
        cb.degrade_faces(gt, with_stages(bare, mask=m, gray=True), in_size=128)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, with_stages(bare, mask=np.zeros((64, 64), np.uint8)), in_size=128)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, with_stages(bare, mask=m.astype(bool)), in_size=128)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, with_stages(chain, mask=m), in_size=128)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, with_stages(bare, gray=True), in_size=64)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, [chain[0], bare[1]], in_size=128)
    for bad in ([('hue', 0.75)], [('brightness', -0.5)], [('saturation', float('nan'))], [('contrast', 0.1)],
                [('hue', 0.05), ('hue', 0.05)], [('gamma', 1.0)]):
        with pytest.raises(ValueError):
            cb.degrade_faces(gt, with_stages(chain, jitter_pt=[bad, bad]), in_size=128)
    with pytest.raises(ValueError):
        cb.degrade_faces(gt, with_stages(chain, jitter=np.zeros(2, F32)), in_size=128)
    with pytest.raises(ValueError):
        DG.sample_degradations(1, gt_size=128, in_size=64, **DG.INPAINTING_OPTIONS)
    lib = cb._lib.load()
    assert lib.cfb_degrade_color_workspace_bytes(1, 128, None, None, None, 64) == -1
