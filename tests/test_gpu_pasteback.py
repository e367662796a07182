"""Whole-image paste-back on the GPU (codeformer_b200.pasteback) against tests/golden/pasteback.npz, which holds the
UNMODIFIED reference FaceRestoreHelper's crops and pastes (oracle/gen_golden_pasteback.py)."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import pasteback_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
pytestmark = pytest.mark.gpu
CASES = {'P1': (2, True), 'P2': (1, False), 'P3': (2, True)}


@pytest.fixture(scope='module')
def gold():
    g = np.load(os.path.join(GOLD, 'pasteback.npz'))
    faces = np.ascontiguousarray(np.load(os.path.join(GOLD, 'faces.npz'))['faces'][..., ::-1])
    return g, faces


def run_case(g, faces, case, debug=False):
    from codeformer_b200 import pasteback as PB
    up, use_parse = CASES[case]
    img_np, up_np, _, _ = O.golden_case(g, faces, case, up)
    img = torch.from_numpy(img_np).cuda()
    restored = np.stack([faces[i] for i in g[f'{case}_faces']])
    if case == 'P3':      # the face upsampler stub of the golden: nearest x2
        restored = np.repeat(np.repeat(restored, 2, axis=1), 2, axis=2)
    restored = torch.from_numpy(np.ascontiguousarray(restored)).cuda()
    n = restored.shape[0]
    masks = None
    if use_parse:
        bits = np.unpackbits(g[f'{case}_parse'])[:n * 512 * 512].reshape(n, 512, 512)
        masks = torch.from_numpy(bits * np.uint8(255)).cuda()
    upsample = None if up_np is None else torch.from_numpy(up_np).cuda()
    inv = PB.adjust_inverse_affines([m.copy() for m in g[f'{case}_inv']], up, case == 'P3')
    return PB._paste(img, restored, inv, up, restored.shape[1], masks, upsample, debug=debug), inv


@pytest.mark.parametrize('mode', ['constant', 'reflect101', 'reflect'])
def test_crops_bit_exact(gold, mode):
    from codeformer_b200 import warp_faces
    g, faces = gold
    img = torch.from_numpy(O.golden_case(g, faces, 'P1', 2)[0]).cuda()
    crop = warp_faces(img, [g['crop_affine']], 512, mode)[0].cpu().numpy()
    assert hashlib.sha256(np.ascontiguousarray(crop).tobytes()).hexdigest() == str(g[f'crop_{mode}_sha256'])


def test_background_resize_bit_exact(gold):
    from codeformer_b200.pasteback import resize_linear
    g, faces = gold
    img = O.golden_case(g, faces, 'P1', 2)[0]
    out = resize_linear(torch.from_numpy(img).cuda(), (img.shape[1] * 2, img.shape[0] * 2)).cpu().numpy()
    assert np.array_equal(out, O.resize_linear_u8(img, (img.shape[1] * 2, img.shape[0] * 2)))
    half = resize_linear(torch.from_numpy(out).cuda(), (img.shape[1], img.shape[0])).cpu().numpy()
    assert np.array_equal(half, O.resize_linear_u8(out, (img.shape[1], img.shape[0])))


@pytest.mark.parametrize('case', list(CASES))
def test_paste_matches_reference(gold, case):
    g, faces = gold
    (out, w_edge, dbg), inv = run_case(g, faces, case, debug=True)
    out, dbg = out.cpu().numpy(), dbg.cpu().numpy()
    assert list(w_edge) == list(g[f'{case}_w_edge'])
    _, _, bg, ref = O.golden_case(g, faces, case, CASES[case][0])
    assert np.array_equal(out, ref), f'{int((out != ref).sum())} values differ from the reference'
    np.testing.assert_allclose(dbg.reshape(-1)[O.sample_index(dbg.size)], g[f'{case}_sample_val'], rtol=0, atol=1e-3)
    # outside every face's ROI the image is the background
    h_up, w_up = ref.shape[:2]
    outside = np.ones((h_up, w_up), bool)
    for m in inv:
        x0, y0, x1, y1 = O.face_roi(m, 512 * (2 if case == 'P3' else 1), h_up, w_up)
        outside[y0:y1, x0:x1] = False
    assert outside.any() and np.array_equal(out[outside], bg[outside])


def test_paste_deterministic(gold):
    g, faces = gold
    (a, _), _ = run_case(g, faces, 'P1')
    (b, _), _ = run_case(g, faces, 'P1')
    assert torch.equal(a, b)


def test_drop_in_matches_device_level(gold):
    """paste_faces_to_input_image on a helper-like object with a parsing module equals the device-level call, and
    edits the helper's inverse affines in place as the reference does."""
    from types import SimpleNamespace
    from codeformer_b200 import init_parsing_model, paste_faces, paste_faces_to_input_image
    from codeformer_b200.parsing import parsenet_spec, random_parsenet_state_dict
    g, faces = gold
    net = init_parsing_model(device='cpu')
    net.load_state_dict(random_parsenet_state_dict(parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=False)
    net = net.cuda()
    img = O.golden_case(g, faces, 'P1', 2)[0]
    inv = [m.copy() for m in g['P1_inv']]
    restored = [faces[i] for i in g['P1_faces']]
    helper = SimpleNamespace(input_img=img, upscale_factor=2, face_size=(512, 512), restored_faces=restored,
                             inverse_affine_matrices=inv, use_parse=True, face_parse=net)
    out = paste_faces_to_input_image(helper)
    dev = paste_faces(torch.from_numpy(img).cuda(), torch.from_numpy(np.stack(restored)).cuda(), g['P1_inv'], 2,
                      face_parse=net).cpu().numpy()
    assert np.array_equal(out, dev)
    for a, b in zip(helper.inverse_affine_matrices, g['P1_inv']):
        np.testing.assert_array_equal(a[:, 2], b[:, 2] + 1.0)


def test_chain_matches_host_crops(gold):
    """warp_faces -> forward_u8 -> paste_faces equals the same chain with host crops through restore_faces."""
    from codeformer_b200 import ARCH_REGISTRY, paste_faces, warp_faces
    from codeformer_b200 import spec as S
    g, faces = gold
    net = ARCH_REGISTRY.get('CodeFormer')(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                                          connect_list=['32', '64', '128', '256']).cuda()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    net = net.eval()
    img = torch.from_numpy(O.golden_case(g, faces, 'P1', 2)[0]).cuda()
    from oracle.pasteback_oracle import invert_affine
    affines = [invert_affine(m / 2.0) for m in g['P1_inv']]
    crops = warp_faces(img, affines)
    with torch.no_grad():
        dev_faces = net.forward_u8(crops, w=0.5)
        host_faces = net.restore_faces(list(crops.cpu().numpy()), w=0.5, on_error='raise')
    host_faces = torch.from_numpy(np.stack(host_faces)).cuda()
    assert torch.equal(dev_faces, host_faces)
    a = paste_faces(img, dev_faces, g['P1_inv'], 2)
    b = paste_faces(img, host_faces, g['P1_inv'], 2)
    assert torch.equal(a, b)


def test_error_cases(gold):
    from types import SimpleNamespace
    from codeformer_b200 import paste_faces, paste_faces_to_input_image, warp_faces
    g, faces = gold
    img = O.golden_case(g, faces, 'P2', 1)[0]
    helper = SimpleNamespace(input_img=img, upscale_factor=1, face_size=(512, 512), restored_faces=[faces[3]],
                             inverse_affine_matrices=[g['P2_inv'][0].copy()], use_parse=False, face_parse=None)
    with pytest.raises(NotImplementedError):
        paste_faces_to_input_image(helper, draw_box=True)
    with pytest.raises(NotImplementedError):
        paste_faces_to_input_image(SimpleNamespace(**{**vars(helper), 'input_img': np.zeros((8, 8, 4), np.uint8)}))
    with pytest.raises(NotImplementedError):
        paste_faces_to_input_image(SimpleNamespace(**{**vars(helper), 'input_img': img.astype(np.uint16)}))
    with pytest.raises(NotImplementedError):
        paste_faces_to_input_image(helper, upsample_img=np.zeros((10, 10, 3), np.uint8))
    with pytest.raises(RuntimeError):
        warp_faces(torch.from_numpy(img), [g['crop_affine']])
    with pytest.raises(RuntimeError):
        paste_faces(torch.from_numpy(img), torch.from_numpy(faces[3:4].copy()), g['P2_inv'][:1], 1)
