"""CPU checks of the restatements behind tests/test_gpu_latent_codes.py: the loop body of scripts/generate_latent_gt.py on the
unmodified reference VQAutoEncoder, cv2's mirror, and the float64 cross-entropy."""
import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from codeformer_b200 import spec as S
from oracle import ref_shim
from oracle.plumbing_oracle import face_to_input
from tests.latent_restate import cross_entropy_f64, feat_mse_f64, script_latent_gt
from tests.util import golden

torch.set_grad_enabled(False)


def test_cv2_flip_is_a_column_reversal():
    rng = np.random.default_rng(0)
    for shape in ((512, 512, 3), (7, 13, 3), (1, 1, 3)):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(cv2.flip(img, 1), img[:, ::-1])
        inplace = img.copy()
        cv2.flip(inplace, 1, inplace)                       # the script flips in place (generate_latent_gt.py:48)
        assert np.array_equal(inplace, img[:, ::-1])


def test_cross_entropy_f64_equals_torch():
    gen = torch.Generator().manual_seed(1)
    for scale, offset in ((1.0, 0.0), (8.0, 0.0), (2.0, 300.0)):
        logits = scale * torch.randn(3, 256, 1024, generator=gen) + offset
        gt = torch.randint(0, 1024, (3, 256), generator=gen)
        ref = F.cross_entropy(logits.double().permute(0, 2, 1), gt, reduction='none').mean(1)
        assert torch.allclose(cross_entropy_f64(logits, gt), ref, rtol=1e-13, atol=0)
    logits[1, 5, 7] = float('nan')
    ce = cross_entropy_f64(logits, gt)
    assert torch.isnan(ce[1]) and torch.isfinite(ce[[0, 2]]).all()


def test_feat_mse_f64_equals_reference_loss():
    """feat_mse is codeformer_idx_model.py:104-107's l_feat_encoder per face (before its weight), in float64."""
    gen = torch.Generator().manual_seed(2)
    E = torch.randn(1024, 256, generator=gen)
    gt = torch.randint(0, 1024, (2, 256), generator=gen)
    lq = torch.randn(2, 256, 16, 16, generator=gen)
    quant = E[gt].view(2, 16, 16, 256).permute(0, 3, 1, 2).double()         # get_codebook_feat(idx, [b,16,16,256])
    ref = torch.stack([torch.mean((quant[i] - lq[i].double()) ** 2) for i in range(2)])
    assert torch.allclose(feat_mse_f64(E, gt, lq), ref, rtol=1e-13, atol=0)


@pytest.mark.skipif(not ref_shim.available(), reason='reference tree not present')
def test_script_restatement_matches_reference_vqautoencoder():
    """The restated loop body on the UNMODIFIED reference VQAutoEncoder (encoder + quantize, seeded weights) picks the oracle's
    codes, for the face and its mirror; and the script's own call encoder(img, True) raises TypeError there."""
    from oracle import codeformer_oracle as O
    _, RefVQ, _, _ = ref_shim.load()
    sd = S.random_state_dict(S.vqae_spec(), 2)
    ref = RefVQ(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', codebook_size=1024).eval()
    ref.load_state_dict(sd, strict=True)
    face = np.ascontiguousarray(golden('faces.npz')['faces'][0][..., ::-1])
    got = script_latent_gt([face], ['00000'], ref, 'cpu')
    assert list(got) == ['orig', 'hflip'] and list(got['orig']) == ['00000']
    for kind, img in (('orig', face), ('hflip', face[:, ::-1])):
        z, _ = O.encoder_forward(sd, torch.from_numpy(face_to_input(np.ascontiguousarray(img)[None])))
        _, _, st = O.vq_forward(sd, z)
        codes = st['min_encoding_indices'].view(16, 16).numpy()
        assert got[kind]['00000'].dtype == np.int64 and np.array_equal(got[kind]['00000'], codes), kind
    with pytest.raises(TypeError):
        ref.encoder(torch.from_numpy(face_to_input(face[None])), True)
