"""gpu: the FID Inception-v3 on the conv engine against the CPU restatement (oracle/fid_oracle.py, pinned to the patched
torchvision model by tests/test_oracle_fid.py): the per-tap engine's explicit windows, the input stage, the pools, the pool3
features, batch invariance, the statistics and the distance against numpy / scipy, sweeps, lists and the errors."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib, fid
from codeformer_b200 import spec as S
from oracle import fid_oracle as fo
from tests.gpu_util import stream
from tests.test_gpu_wholeimage import nets, whole_images   # noqa: F401  (nets: fixture)

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
CONV_BAR = 6e-5          # x max|ref|, the per-tap bar of test_gpu_detection (split-fp16 operands, fp32 accumulation)
# pool3 against the fp32 oracle, x max|feature|: 93 split-fp16 convs.  Measured on an H100: 3.4e-5 .. 3.6e-5 at B = 1 and 3
# for 299^2, 512^2 faces and 64 x 96 (the test prints it); the bar leaves a factor ~3
FEAT_BAR = 1e-4
OUT_RELU = 3               # cfb::OUT_RELU


@pytest.fixture(scope='module')
def sd():
    return fo.random_fid_state_dict(1)


@pytest.fixture(scope='module')
def net(sd):
    n = cb.InceptionV3().to(DEV)
    n.load_state_dict(sd, strict=True)
    return n


def _faces(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(n, 3, h // 8 + 1, w // 8 + 1, generator=g), size=(h, w), mode='bilinear', align_corners=False)
    x = (base * 200 + 40 * torch.rand(n, 3, h, w, generator=g)).round().clamp(0, 255)
    return x.permute(0, 2, 3, 1).to(torch.uint8).contiguous()


FORMS = [(1, 7, 0, 3, 1), (7, 1, 3, 0, 1), (1, 3, 0, 1, 1), (3, 1, 1, 0, 1), (5, 5, 2, 2, 1), (3, 3, 0, 0, 1), (3, 3, 0, 0, 2),
         (1, 1, 0, 0, 1)]


# every form at the odd sizes of the network; 299 (the stem input) with the valid 3x3 forms only
CASES = [(f, n) for n in (35, 17, 147) for f in FORMS] + [(f, 299) for f in FORMS if f[:2] == (3, 3) and f[2] == 0]


@pytest.mark.parametrize('form,size', CASES, ids=lambda v: '{}x{}p{}{}s{}'.format(*v) if isinstance(v, tuple) else str(v))
def test_window_conv_forms(form, size):
    kh, kw, ph, pw, s = form
    lib = _lib.load()
    g = torch.Generator().manual_seed(size * 10 + kh)
    N, cin, cout, pitch, c0 = 2, 64 if size >= 147 else 192, 96 if size < 147 else 32, 256, 100
    x = torch.randn(N, cin, size, size + 2, generator=g)
    w = torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    ref = F.relu(F.conv2d(x, w, b, stride=s, padding=(ph, pw)))
    ho, wo = ref.shape[2], ref.shape[3]
    fill = torch.full((N, ho, wo, pitch), 7.0, device=DEV)
    xin = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    need = lib.cfb_conv2d_pertap_window_workspace_bytes(N, size, size + 2, cin, cout, kh, kw, s, ph, pw)
    ws = torch.empty(int(need), dtype=torch.uint8, device=DEV)
    wd, bd = w.to(DEV), b.to(DEV)      # kept alive until the launch has read them
    _lib.check(lib.cfb_conv2d_pertap_window_nhwc(_lib.ptr(xin), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(fill), N, size,
                                                  size + 2, cin, cout, kh, kw, s, ph, pw, OUT_RELU, pitch, c0, _lib.ptr(ws), need,
                                                  stream()),
               'cfb_conv2d_pertap_window_nhwc')
    got = fill[..., c0:c0 + cout].permute(0, 3, 1, 2).cpu()
    err = (got - ref).abs().max().item()
    assert err <= CONV_BAR * ref.abs().max().item(), err
    assert bool((fill[..., :c0] == 7).all()) and bool((fill[..., c0 + cout:] == 7).all())


@pytest.mark.parametrize('size', [(512, 512), (64, 96), (299, 299), (37, 300)])
@pytest.mark.parametrize('normalize', [False, True])
def test_input_stage(size, normalize):
    H, W = size
    u8 = _faces(2, H, W, H + W)
    x = fo.u8_to_tensor(u8)
    want = fo.input_stage(x, True, normalize)
    assert torch.equal(fid.fid_input(u8.to(DEV), True, normalize).cpu(), want)
    assert torch.equal(fid.fid_input(x.to(DEV), True, normalize).cpu(), want)
    xr = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(3))
    assert torch.equal(fid.fid_input(xr.to(DEV), True, normalize).cpu(), fo.input_stage(xr, True, normalize))
    assert torch.equal(fid.fid_input(xr.to(DEV), False, normalize).cpu(), fo.input_stage(xr, False, normalize))


@pytest.mark.parametrize('kind', [0, 1, 2])
@pytest.mark.parametrize('hw', [(35, 35), (17, 17), (147, 147), (8, 9)])
def test_pools(kind, hw):
    """max pools bit-equal to torch; avg pool (count_include_pad=False) bit-equal as well, the bar allows one ulp"""
    H, W = hw
    g = torch.Generator().manual_seed(H * 3 + kind)
    x = F.relu(torch.randn(2, 64, H, W, generator=g))
    x[0, 3, 1, 1] = float('nan')
    if kind == 0:
        want = F.max_pool2d(x, 3, 2)
    elif kind == 1:
        want = F.max_pool2d(x, 3, 1, 1)
    else:
        want = F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
    xin = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.empty((2, want.shape[2], want.shape[3], 64), device=DEV)
    _lib.check(_lib.load().cfb_debug_fid_pool(_lib.ptr(xin), _lib.ptr(out), 2, H, W, 64, kind, stream()), 'cfb_debug_fid_pool')
    got = out.permute(0, 3, 1, 2).cpu()
    if kind < 2:
        assert torch.equal(torch.isnan(got), torch.isnan(want)) and bool(torch.isnan(want).any())
        assert torch.equal(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(want, nan=-1.0))
    else:
        ok = torch.isnan(want)
        assert torch.equal(torch.isnan(got), ok)
        ulp = torch.nextafter(want.abs(), torch.tensor(float('inf'))) - want.abs()
        assert bool(((got - want).abs()[~ok] <= ulp[~ok]).all())
        print('avg pool values off by one ulp:', int(((got != want) & ~ok).sum()))


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('case', ['299', 'face512', '64x96'])
def test_features_vs_oracle(net, sd, B, case):
    if case == '299':
        x = torch.rand(B, 3, 299, 299, generator=torch.Generator().manual_seed(B)) * 2 - 1
        net.resize_input, net.normalize_input = False, False
        try:
            got = net(x.to(DEV))[0].view(B, -1).cpu()
        finally:
            net.resize_input, net.normalize_input = True, True
        want = fo.forward(sd, x, False, False).view(B, -1)
    else:
        H, W = (512, 512) if case == 'face512' else (64, 96)
        u8 = _faces(B, H, W, B + H)
        got = net.forward_u8(u8.to(DEV)).cpu()
        want = fo.forward(sd, fo.u8_to_tensor(u8)).view(B, -1)
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    print(f'pool3 {case} B={B}: max err {err:.3e}, max |feature| {scale:.3e}, ratio {err / scale:.3e}')
    assert err <= FEAT_BAR * scale


def test_forward_u8_equals_unfused_chain(net):
    u8 = _faces(3, 512, 512, 9).to(DEV)
    x = fid.fid_input(u8, True, True)
    net.resize_input, net.normalize_input = False, False
    try:
        chain = net(x)[0].view(3, -1)
    finally:
        net.resize_input, net.normalize_input = True, True
    assert torch.equal(net.forward_u8(u8), chain)


def test_batch_invariance_and_repeats(net):
    u8 = _faces(32, 128, 128, 11).to(DEV)
    full = net.forward_u8(u8)
    assert torch.equal(net.forward_u8(u8), full)
    for mb in (1, 4):
        assert torch.equal(cb.inception_features(u8, net, max_batch=mb), full)
    assert torch.equal(net.forward_u8(u8[5:8]), full[5:8])
    assert torch.equal(net.forward_u8(u8[17:18]), full[17:18])
    # statistics of features computed one image per launch equal those of one launch for all 32
    one = torch.cat([net.forward_u8(u8[i:i + 1]) for i in range(32)])
    mu, sigma = cb.fid_statistics(full)
    m1, s1 = cb.fid_statistics(one)
    assert torch.equal(m1, mu) and torch.equal(s1, sigma)


def test_statistics_vs_numpy():
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(500, 2048, generator=g) * torch.rand(2048, generator=g) * 3 + 5 * torch.rand(2048, generator=g))
    mu, sigma = cb.fid_statistics(x.to(DEV))
    xn = x.double().numpy()
    mu_ref, sig_ref = np.mean(xn, axis=0), np.cov(xn, rowvar=False)
    assert np.abs(mu.cpu().numpy() - mu_ref).max() <= 1e-12 * np.abs(mu_ref).max()
    assert np.abs(sigma.cpu().numpy() - sig_ref).max() <= 1e-12 * np.abs(sig_ref).max()
    assert torch.equal(sigma, sigma.T)
    # a repeated call gives the same bits, and so does a feature matrix at an address that is not 16-byte aligned (copied)
    m2, s2 = cb.fid_statistics(x.to(DEV))
    assert torch.equal(m2, mu) and torch.equal(s2, sigma)
    buf = torch.empty(500 * 2048 + 1, device=DEV)
    buf[1:] = x.to(DEV).view(-1)
    m3, s3 = cb.fid_statistics(buf[1:].view(500, 2048))
    assert torch.equal(m3, mu) and torch.equal(s3, sigma)


def _random_cov_features(n, d, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(d, d)) / np.sqrt(d)
    z = rng.normal(size=(n, d))
    return (scale * z @ a + rng.normal(size=d)).astype(np.float32)


def test_frechet_distance_full_rank():
    xa = _random_cov_features(4096, 2048, 1)
    xb = _random_cov_features(4096, 2048, 2, 1.2)
    sa, sb = cb.fid_statistics(torch.from_numpy(xa).to(DEV)), cb.fid_statistics(torch.from_numpy(xb).to(DEV))
    got = cb.frechet_distance(sa, sb)
    want = cb.calculate_fid(sa[0].cpu().numpy(), sa[1].cpu().numpy(), sb[0].cpu().numpy(), sb[1].cpu().numpy())
    print('full-rank FID', got, want)
    assert abs(got - want) <= 1e-6 * abs(want)
    # identical sets
    same = cb.frechet_distance(sa, sa)
    assert abs(same) <= 1e-6 * float(torch.trace(sa[1]))


def test_frechet_distance_rank_deficient():
    """N = 100 features in 2048 dimensions: both covariances have rank 99, so sigma_a sigma_b has ~1950 zero eigenvalues.
    sqrtm and the eigendecomposition each turn those zeros into roundoff of order 1e-16 * |sigma|^2 whose square roots add up to
    ~2048 * 1e-8 * |sigma|: the two traces can differ by that much, far above 1e-6 relative only when FID itself is tiny.  The bar
    is 1e-4 relative to FID."""
    xa = _random_cov_features(100, 2048, 3)
    xb = _random_cov_features(100, 2048, 4, 1.5)
    sa, sb = cb.fid_statistics(torch.from_numpy(xa).to(DEV)), cb.fid_statistics(torch.from_numpy(xb).to(DEV))
    got = cb.frechet_distance(sa, sb)
    want = cb.calculate_fid(sa[0].cpu().numpy(), sa[1].cpu().numpy(), sb[0].cpu().numpy(), sb[1].cpu().numpy())
    print('rank-deficient FID', got, want)
    assert abs(got - want) <= 1e-4 * abs(want)


def test_real_fidelity_sweep(net):
    faces = torch.from_numpy(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'faces.npz'))['faces'][:2]).to(DEV)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    sweep = cf.forward_u8_sweep(faces, [0.0, 0.5, 1.0])
    feats = cb.inception_features(sweep, net)
    assert feats.shape == (3, 2, 2048)
    ref = cb.fid_statistics(cb.inception_features(faces, net))
    scores = cb.fid_scores(sweep, ref, net)
    assert scores.shape == (3,)
    for k in range(3):
        fk = cb.inception_features(sweep[:, k].contiguous(), net)
        assert torch.equal(feats[k], fk)
        mk, sk = cb.fid_statistics(fk)
        m2, s2 = cb.fid_statistics(feats[k])
        assert torch.equal(mk, m2) and torch.equal(sk, s2)
        assert float(scores[k]) == cb.frechet_distance((mk, sk), ref)
    print('sweep FID', scores.numpy())


def test_lists_restored_images(net, nets):   # noqa: F811
    imgs = whole_images()[:3]
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser)
    feats = cb.inception_features(res, net)
    assert feats.shape == (len(res), 2048)
    for i, r in enumerate(res):
        r = r if torch.is_tensor(r) else torch.from_numpy(r).to(DEV)
        assert torch.equal(feats[i], net.forward_u8(r[None].to(DEV))[0])
    rng = np.random.default_rng(5)
    mixed = [rng.integers(0, 256, s).astype(np.uint8) for s in [(40, 56, 3), (80, 80, 3), (40, 56, 3)]]
    fm = cb.inception_features(mixed, net)
    for i, m in enumerate(mixed):
        assert torch.equal(fm[i], net.forward_u8(torch.from_numpy(m)[None].to(DEV))[0])
    cb.check_async_status()


def test_errors_and_nan(net):
    u8 = _faces(2, 64, 64, 50)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        net(fo.u8_to_tensor(u8))
    with pytest.raises(RuntimeError):
        net(fo.u8_to_tensor(u8).double().to(DEV))
    with pytest.raises(RuntimeError):
        net(fo.u8_to_tensor(u8)[:, :2].to(DEV))
    with pytest.raises(NotImplementedError):
        net.forward_u8(u8.float().to(DEV))
    with pytest.raises(RuntimeError):
        net.forward_u8(u8[..., :2].contiguous().to(DEV))
    with pytest.raises(NotImplementedError):
        cb.inception_features([u8[0].numpy().astype(np.uint16)], net)
    with pytest.raises(ValueError):
        cb.inception_features(u8[0].to(DEV), net)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.fid_statistics(torch.rand(4, 64))
    with pytest.raises(RuntimeError):
        cb.fid_statistics(torch.rand(4, 64, device=DEV).double())
    with pytest.raises(ValueError, match='at least 2'):
        cb.fid_statistics(torch.rand(1, 2048, device=DEV))
    with pytest.raises(ValueError):
        cb.fid_statistics(torch.rand(4, 100, device=DEV))
    for kw in ({'output_blocks': (2,)}, {'use_fid_inception': False}, {'requires_grad': True}):
        with pytest.raises(NotImplementedError):
            cb.InceptionV3(**kw)
    # NaN input: NaN features for that image, as torch gives, no fault, and the other image of the batch is unaffected
    x = fo.u8_to_tensor(u8)
    x[0, 1, 5, 7] = float('nan')
    out = net(x.to(DEV))[0].view(2, -1)
    torch.cuda.synchronize()
    assert torch.isnan(out[0]).all() and torch.isfinite(out[1]).all()
    assert torch.equal(out[1], net(x[1:].to(DEV))[0].view(1, -1)[0])
    assert torch.isnan(fo.forward(fo.random_fid_state_dict(1), x[:1])).all()
    # also without the resize, and for a NaN in the last row and column the first conv reads
    y = torch.rand(2, 3, 299, 299, generator=torch.Generator().manual_seed(6)) * 2 - 1
    y[1, 2, 298, 298] = float('nan')
    net.resize_input, net.normalize_input = False, False
    try:
        out = net(y.to(DEV))[0].view(2, -1)
    finally:
        net.resize_input, net.normalize_input = True, True
    assert torch.isfinite(out[0]).all() and torch.isnan(out[1]).all()
    cb.check_async_status()
