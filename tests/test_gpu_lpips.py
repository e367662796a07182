"""gpu: LPIPS-VGG on the conv engine against the CPU restatement (oracle/lpips_oracle.py, pinned to torchvision and the
reference's LPIPSLoss by tests/test_oracle_lpips.py): the stem and the fused head-and-pool pass against torch, forward,
the uint8 conventions, batch and sweep invariance, lists of whole images, LPIPSLoss and the errors."""
import ctypes
import os

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from oracle import lpips_oracle as LO
from tests.test_gpu_wholeimage import nets, whole_images   # noqa: F401  (nets: fixture)

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
# forward against the fp32 oracle, relative to the value (split-fp16 operands on 12 of the 13 convs)
VAL_BAR = 1e-4
HEAD_BAR = 1e-6


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope='module')
def sd():
    return LO.random_lpips_state_dict(1)


@pytest.fixture(scope='module')
def net(sd):
    n = cb.LPIPS().to(DEV)
    n.load_state_dict(sd, strict=True)
    return n


@pytest.fixture(scope='module')
def oracle(sd):
    lp = LO.LPIPS()
    lp.load_state_dict(sd, strict=True)
    return lp


def _images(n, h, w, seed, noise=0.2):
    """Seeded uint8 BGR images with smooth structure, and candidates that differ by noise."""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(n, 3, h // 8 + 1, w // 8 + 1, generator=g), size=(h, w), mode='bilinear', align_corners=False)
    ref = (base * 255).round().clamp(0, 255)
    cand = (ref + noise * 255 * (torch.rand(ref.shape, generator=g) - 0.5)).round().clamp(0, 255)
    to = lambda t: t.permute(0, 2, 3, 1).to(torch.uint8).contiguous()       # noqa: E731
    return to(ref), to(cand)


def _f32(u8):
    """uint8 BGR [N,H,W,3] -> fp32 RGB [N,3,H,W] in [-1, 1] (lpips.im2tensor)."""
    return torch.cat([LO.im2tensor(np.ascontiguousarray(x[:, :, ::-1])) for x in u8.cpu().numpy()])


def _rel(a, b):
    return float(((a - b).abs() / b.abs().clamp_min(1e-12)).max())


# ---- kernels against torch -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('u8', [False, True], ids=['f32', 'u8'])
def test_stem(net, sd, u8):
    lib = _lib.load()
    B, G, H, W = 2, 2, 20, 150
    ref8, _ = _images(B, H, W, 1)
    cand8, _ = _images(B * G, H, W, 2)
    net._prepare(torch.device(DEV))
    modes = [0, 1, 2, 4, 6] if not u8 else [0, 1]
    for mode in modes:
        out = torch.empty((B * (1 + G), H, W, 64), device=DEV)
        if u8:
            a, b = ref8.to(DEV), cand8.to(DEV)
            conv = 'lpips' if mode == 0 else 'codeformer'
            x = torch.cat([LO.stem_input(im, conv) for im in torch.cat([ref8, cand8]).cpu().numpy()])
        else:
            a, b = _f32(ref8).to(DEV), (_f32(cand8) * 0.9).to(DEV)
            x = torch.cat([a, b]).cpu()
            if mode & 2:
                x = (x + 1) / 2
            if mode & 4:
                x = (x - torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)) / torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
            if mode & 1:
                x = 2 * x - 1
            x = LO.ScalingLayer()(x)
        assert lib.cfb_debug_lpips_stem(net._net, _lib.ptr(a), _lib.ptr(b), int(u8), mode, _lib.ptr(out), B, H, W, G, _stream()) == 0
        # launch order: group q = [ref q, cand q*G .. q*G+G-1]
        order = [i for q in range(B) for i in [q] + [B + q * G + j for j in range(G)]]
        ref = F.relu(F.conv2d(x[order], sd['net.slice1.0.weight'], sd['net.slice1.0.bias'], padding=1)).permute(0, 2, 3, 1)
        err = float((out.cpu() - ref).abs().max())
        assert err <= 1e-5 * max(1.0, float(ref.abs().max())), (mode, err)


@pytest.mark.parametrize('C,H,W,G', [(64, 34, 47, 1), (128, 16, 16, 3), (256, 9, 12, 2), (512, 5, 3, 4), (512, 1, 1, 1)])
def test_head_and_pool(C, H, W, G):
    lib = _lib.load()
    B = 3
    g = torch.Generator().manual_seed(C + H)
    feat = torch.relu(torch.randn(B * (1 + G), H, W, C, generator=g))
    feat[0, 0, 0, :5] = float('nan') if C == 128 else feat[0, 0, 0, :5]
    lin = torch.rand(C, generator=g) / C
    pooled = torch.empty((B * (1 + G), H // 2, W // 2, C), device=DEV)
    res = torch.empty(B * G, device=DEV)
    need = lib.cfb_debug_lpips_head_workspace_bytes(B, H, W, G)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    fd, ld = feat.to(DEV), lin.to(DEV)
    assert lib.cfb_debug_lpips_head(_lib.ptr(fd), _lib.ptr(ld), _lib.ptr(pooled) if H > 1 else None, _lib.ptr(res), B, H, W, G, C,
                                    _lib.ptr(ws), need, _stream()) == 0
    x = feat.permute(0, 3, 1, 2)
    if H > 1:
        pool_ref = F.max_pool2d(x.to(DEV), 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(torch.isnan(pooled), torch.isnan(pool_ref))
        assert torch.equal(torch.nan_to_num(pooled), torch.nan_to_num(pool_ref))
    xd = x.double()
    nf = xd / (torch.sqrt((xd ** 2).sum(1, keepdim=True)) + 1e-10)
    ref = []
    for q in range(B):
        for j in range(G):
            d = (nf[q * (1 + G)] - nf[q * (1 + G) + 1 + j]) ** 2
            ref.append(float((d * lin.double().view(C, 1, 1)).sum(0).mean()))
    ref = torch.tensor(ref, dtype=torch.float64)
    out = res.cpu().double()
    if C == 128:       # the NaN pixel poisons the first group's values only
        assert torch.isnan(out[:G]).all() and torch.isfinite(out[G:]).all()
        out, ref = out[G:], ref[G:]
    assert _rel(out, ref) <= HEAD_BAR, _rel(out, ref)


# ---- the network ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', [(1, 64, 96), (3, 64, 96), (1, 224, 224), (1, 512, 512)])
def test_forward_vs_oracle(net, oracle, shape):
    N, H, W = shape
    r8, c8 = _images(N, H, W, H + N)
    a, b = _f32(r8), _f32(c8)
    out, layers = net(a.to(DEV), b.to(DEV), retPerLayer=True)
    with torch.no_grad():
        ref, ref_layers = oracle(a, b, retPerLayer=True)
    assert out.shape == (N, 1, 1, 1) and len(layers) == 5
    err = _rel(out.cpu().double(), ref.double())
    # per layer: the error against the total (a deep layer's value can be small next to it)
    lerr = [float(((layers[k].cpu().double() - ref_layers[k].double()).abs() / ref.double().abs()).max()) for k in range(5)]
    print(f'forward {shape}: max relative error {err:.2e} (per layer, of the total: {[f"{e:.1e}" for e in lerr]}), '
          f'values {ref.flatten().tolist()}')
    assert err <= VAL_BAR
    assert max(lerr) <= VAL_BAR
    # retPerLayer is consistent with val: the layers summed in order 0..4 in float32
    s = layers[0].clone()
    for k in range(1, 5):
        s += layers[k]
    assert torch.equal(s, out)
    assert torch.equal(net(a.to(DEV), b.to(DEV), normalize=False), out)
    # normalize=True maps [0, 1] inputs to [-1, 1] first
    o2 = net(((a + 1) / 2).to(DEV), ((b + 1) / 2).to(DEV), normalize=True)
    assert _rel(o2.cpu().double(), oracle((a + 1) / 2, (b + 1) / 2, normalize=True).double()) <= VAL_BAR


def test_identical_inputs_give_zero(net):
    r8, _ = _images(2, 48, 64, 3)
    a = _f32(r8).to(DEV)
    assert torch.equal(net(a, a.clone()), torch.zeros(2, 1, 1, 1, device=DEV))
    assert torch.equal(net.forward_u8(r8.to(DEV), r8.to(DEV)), torch.zeros(2, device=DEV))


@pytest.mark.parametrize('convention', ['lpips', 'codeformer'])
def test_forward_u8_equals_unfused_chain(net, convention):
    r8, c8 = _images(3, 64, 96, 11)
    r8, c8 = r8.to(DEV), c8.to(DEV)
    got = net.forward_u8(r8, c8, convention)
    a = torch.cat([LO.input_tensor(x, convention) for x in r8.cpu().numpy()]).to(DEV)
    b = torch.cat([LO.input_tensor(x, convention) for x in c8.cpu().numpy()]).to(DEV)
    if convention == 'lpips':
        want = net(a, b).view(-1)
    else:
        loss = cb.LPIPSLoss(use_input_norm=True, range_norm=True)
        loss.perceptual = net
        want = torch.stack([loss(b[i:i + 1], a[i:i + 1]) for i in range(3)])
    assert torch.equal(got, want)


def test_oracle_u8_distance(net, oracle):
    r8, c8 = _images(1, 64, 96, 12)
    for conv in ('lpips', 'codeformer'):
        got = float(net.forward_u8(r8.to(DEV), c8.to(DEV), conv))
        ref = float(LO.distance_u8(oracle, r8[0].numpy(), c8[0].numpy(), conv))
        assert abs(got - ref) <= VAL_BAR * abs(ref), (conv, got, ref)


def test_batch_invariance_and_repeats(net):
    r8, c8 = _images(32, 64, 96, 13)
    a, b = _f32(r8).to(DEV), _f32(c8).to(DEV)
    full = net(a, b)
    assert torch.equal(net(a[5:6], b[5:6]), full[5:6])
    assert torch.equal(net(a[4:7], b[4:7]), full[4:7])
    assert torch.equal(net(a, b), full)
    u = net.forward_u8(r8.to(DEV), c8.to(DEV))
    for mb in (1, 4):
        assert torch.equal(net.forward_u8(r8.to(DEV), c8.to(DEV), max_batch=mb), u)
    assert torch.equal(cb.lpips_distance(c8.to(DEV), r8.to(DEV), net, max_batch=1), u)


@pytest.mark.parametrize('B,K', [(1, 1), (1, 4), (3, 1), (3, 4)])
def test_sweep_equals_pairs(net, B, K):
    r8, _ = _images(B, 64, 96, 20 + B)
    cands = torch.stack([_images(B, 64, 96, 30 + k)[1] for k in range(K)], 1).to(DEV)     # [B,K,H,W,3]
    r8 = r8.to(DEV)
    got = cb.lpips_distance(cands, r8, net)
    assert got.shape == (B, K)
    assert net.last_launch_images == [B * (1 + K)]        # every reference once, with its K candidates
    for k in range(K):
        assert torch.equal(got[:, k], cb.lpips_distance(cands[:, k].contiguous(), r8, net))
    for mb in (1, 2):
        assert torch.equal(cb.lpips_distance(cands, r8, net, max_batch=mb), got)


def test_real_fidelity_sweep(net):
    faces = torch.from_numpy(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'faces.npz'))['faces'][:2]).to(DEV)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    sweep = cf.forward_u8_sweep(faces, [0.0, 0.5, 1.0])
    d = cb.lpips_distance(sweep, faces, net)
    assert d.shape == (2, 3) and bool(torch.isfinite(d).all())
    assert sum(net.last_launch_images) == 2 + 2 * 3
    for k in range(3):
        assert torch.equal(d[:, k], cb.lpips_distance(sweep[:, k].contiguous(), faces, net))
    print('sweep lpips', d.cpu().numpy())


def test_lists_mixed_sizes(net):
    rng = np.random.default_rng(5)
    refs = [rng.integers(0, 256, s).astype(np.uint8) for s in [(40, 56, 3), (64, 64, 3), (40, 56, 3), (17, 300, 3)]]
    rows = [[np.clip(r.astype(np.int32) + rng.integers(-30, 31, r.shape), 0, 255).astype(np.uint8) for r in refs] for _ in range(3)]
    rows[1] = [torch.from_numpy(x).to(DEV) for x in rows[1]]
    d = cb.lpips_distance(rows[0], refs, net)
    assert d.shape == (4,)
    pairs = [float(net.forward_u8(torch.from_numpy(r)[None].to(DEV), torch.from_numpy(c)[None].to(DEV))) for r, c in zip(refs, rows[0])]
    assert d.cpu().tolist() == pairs
    dk = cb.lpips_distance(rows, refs, net, convention='codeformer')
    assert dk.shape == (3, 4)
    for k in range(3):
        assert torch.equal(dk[k], cb.lpips_distance(rows[k], refs, net, convention='codeformer'))


def test_lists_restored_images(net, nets):   # noqa: F811
    imgs = whole_images()[:3]
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser)
    sweep = cb.restore_images_sweep(imgs, nets.net, nets.det, [0.3, 0.8], parser=nets.parser)
    gts = [cv2.resize(im, (r.shape[1], r.shape[0]), interpolation=cv2.INTER_CUBIC) for im, r in zip(imgs, res)]
    d = cb.lpips_distance(res, gts, net)
    for i, (r, g) in enumerate(zip(res, gts)):
        r = r if torch.is_tensor(r) else torch.from_numpy(r).to(DEV)
        assert float(d[i]) == float(net.forward_u8(torch.from_numpy(g)[None].to(DEV), r[None]))
    dk = cb.lpips_distance(sweep, gts, net)
    assert dk.shape == (2, len(imgs))
    assert torch.equal(dk[1], cb.lpips_distance(sweep[1], gts, net))
    cb.check_async_status()


@pytest.mark.parametrize('range_norm', [False, True])
@pytest.mark.parametrize('use_input_norm', [False, True])
def test_lpips_loss(sd, oracle, range_norm, use_input_norm):
    loss = cb.LPIPSLoss(loss_weight=0.5, use_input_norm=use_input_norm, range_norm=range_norm).to(DEV)
    loss.perceptual.load_state_dict(sd, strict=True)
    ref = LO.LPIPSLoss(loss_weight=0.5, use_input_norm=use_input_norm, range_norm=range_norm)
    ref.perceptual = oracle
    r8, c8 = _images(2, 64, 96, 40)
    pred, target = _f32(c8), _f32(r8)
    got = loss(pred.to(DEV), target.to(DEV))
    want = ref(pred, target)
    assert got.shape == () and abs(float(got) - float(want)) <= VAL_BAR * abs(float(want))
    with torch.enable_grad():
        with pytest.raises(RuntimeError, match='no backward'):
            loss(pred.to(DEV).requires_grad_(), target.to(DEV))


def test_errors_and_nan(net):
    r8, c8 = _images(2, 32, 32, 50)
    a, b = _f32(r8), _f32(c8)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        net(a, b)
    with pytest.raises(RuntimeError):
        net(a.to(DEV), b[:1].to(DEV))
    with pytest.raises(RuntimeError):
        net(a.to(DEV).double(), b.to(DEV).double())
    with pytest.raises(ValueError, match='16'):
        net(a[:, :, :15].to(DEV), b[:, :, :15].to(DEV))
    with pytest.raises(ValueError, match='16'):
        cb.lpips_distance(c8[:, :8].to(DEV), r8[:, :8].to(DEV), net)
    with pytest.raises(NotImplementedError):
        cb.lpips_distance(c8.to(DEV).float(), r8.to(DEV).float(), net)
    with pytest.raises(NotImplementedError):
        cb.lpips_distance([c8[0].numpy().astype(np.uint16)], [r8[0].numpy().astype(np.uint16)], net)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        cb.lpips_distance(c8, r8, net)
    with pytest.raises(ValueError):
        cb.lpips_distance(c8.to(DEV), r8[:1].to(DEV), net)
    with pytest.raises(ValueError):
        cb.lpips_distance([c8[0].numpy()], [r8[0].numpy(), r8[1].numpy()], net)
    with pytest.raises(ValueError):
        net.forward_u8(r8.to(DEV), c8.to(DEV), convention='other')
    # NaN input: NaN values, no fault
    a[0, 1, 5, 7] = float('nan')
    out = net(a.to(DEV), b.to(DEV))
    torch.cuda.synchronize()
    assert torch.isnan(out[0]).all() and torch.isfinite(out[1]).all()
    cb.check_async_status()
