"""CPU: the restatements the aligned-face GPU tests compare against (tests/aligned_restate.py, oracle/plumbing_oracle.py) are
the reference's own arithmetic -- the inpainting script's mask, blend and tensor2img, and the --has_aligned gray test --
checked against img2tensor / normalize / tensor2img (basicsr/utils/img_util.py) and facelib's is_gray."""
import numpy as np
import pytest
import torch

from oracle import plumbing_oracle as P
from oracle import ref_shim
from tests.aligned_restate import aligned_crop, inpaint_blend, inpaint_mask

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.skipif(not ref_shim.available(), reason='reference tree not present')


@pytest.fixture(scope='module')
def ref():
    from oracle.gen_golden_pasteback import load_helper_class
    _, helper_mod = load_helper_class()
    ref_shim.load()
    from basicsr.utils import img2tensor, tensor2img
    from torchvision.transforms.functional import normalize

    def to_input(face):                           # inference_inpainting.py:63-65
        t = img2tensor(face / 255., bgr2rgb=True, float32=True)
        normalize(t, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5), inplace=True)
        return t.unsqueeze(0)

    def script_mask(x):                           # :68-71, for any H x W
        h, w = x.shape[2:]
        mask = torch.zeros(h, w)
        m_ind = torch.sum(x[0], dim=0)
        mask[m_ind == 3] = 1.0
        return mask.view(1, 1, h, w)

    def script_save(x, out):                      # :74-75 and the astype of :82
        mask = script_mask(x)
        output = (1 - mask) * x + mask * out
        return tensor2img(output, rgb2bgr=True, min_max=(-1, 1)).astype('uint8')
    return to_input, script_mask, script_save, helper_mod.is_gray


def _face_with_holes(seed, h=64, w=80):
    rng = np.random.default_rng(seed)
    face = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    face[5:20, 10:40] = 255                                        # a painted block
    face[30, 50] = 255                                             # an isolated white pixel ...
    face[30, 51] = (255, 255, 254)                                 # ... next to near-white ones, in every channel
    face[30, 52] = (255, 254, 255)
    face[30, 53] = (254, 255, 255)
    face[40:44, 60:64] = (255, 255, 255)
    return face


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_inpaint_blend_and_tensor2img_match_the_script(ref, seed):
    to_input, script_mask, script_save, _ = ref
    face = _face_with_holes(seed)
    x = to_input(face)
    assert torch.equal(x, torch.from_numpy(P.face_to_input(face[None])))
    out = torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)) * 0.8    # beyond +-1 too: the clamp
    mask = inpaint_mask(x)
    assert torch.equal(mask, script_mask(x))
    assert int(mask.sum()) == 15 * 30 + 1 + 16
    want = script_save(x, out)
    got = P.output_to_face(inpaint_blend(x, out).numpy())[0]
    assert np.array_equal(got, want)
    # outside the mask the saved face is the input face itself, inside it is tensor2img of the network output
    m = mask[0, 0].numpy().astype(bool)
    assert np.array_equal(got[~m], face[~m])
    assert np.array_equal(got[m], P.output_to_face(out.numpy())[0][m])


def test_inpaint_mask_on_every_byte_triple(ref):
    """All 256^3 (B, G, R) triples through the script's own img2tensor / normalize / sum: only (255, 255, 255) reaches 3, and
    the restated mask agrees everywhere."""
    to_input, script_mask, _, _ = ref
    g, r = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing='ij')
    hits = []
    for b in range(256):
        face = np.stack([np.full_like(g, b), g, r], axis=-1)
        x = to_input(face)
        m = script_mask(x)
        assert torch.equal(inpaint_mask(x), m)
        for gi, ri in zip(*np.nonzero(m[0, 0].numpy())):
            hits.append((b, int(g[gi, ri]), int(r[gi, ri])))
    assert hits == [(255, 255, 255)]


@pytest.mark.parametrize('size', [(512, 512), (256, 256), (1024, 1024), (400, 300), (513, 511)])
def test_aligned_gray_test_matches_facelib(ref, size):
    """The --has_aligned branch's resize and is_gray: the package's host is_gray equals facelib's on gray, near-gray and
    colour crops of every size the GPU tests use."""
    _, _, _, ref_is_gray = ref
    w, h = size
    rng = np.random.default_rng(w * 31 + h)
    base = rng.integers(0, 256, (h, w), dtype=np.uint8)
    gray = np.repeat(base[:, :, None], 3, axis=2)
    near = gray.astype(np.int16) + rng.integers(-4, 5, (h, w, 3))
    near = np.clip(near, 0, 255).astype(np.uint8)
    colour = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    for img in (gray, near, colour):
        crop, flag = aligned_crop(img)
        assert np.array_equal(crop, cv2.resize(img, (512, 512), interpolation=cv2.INTER_LINEAR))
        assert flag == bool(ref_is_gray(crop, threshold=10))
    assert aligned_crop(gray)[1] and not aligned_crop(colour)[1]


def test_gray_moments_decide_as_numpy():
    """The decision restore_images / restore_aligned take from cfb_is_gray_u8's integer sums equals numpy's variances on
    crops that straddle the threshold (a spread of 1-2 levels per channel difference)."""
    from codeformer_b200.wholeimage import is_gray
    for seed in range(20):
        rng = np.random.default_rng(seed)
        base = rng.integers(20, 230, (64, 64), dtype=np.int16)
        img = np.stack([base, base + rng.integers(-4 - seed // 4, 5 + seed // 4, base.shape), base], -1).astype(np.uint8)
        n = img.shape[0] * img.shape[1]
        c = img.astype(np.int64)
        total = 0.0
        for a, b in ((0, 1), (1, 2), (2, 0)):
            d = c[:, :, a] - c[:, :, b]
            s, s2 = int(d.sum()), int((d * d).sum())
            total += (n * s2 - s * s) / (n * n)
        assert (total / 3.0 <= 10) == is_gray(img)
