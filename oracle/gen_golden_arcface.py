"""Write tests/golden/arcface.npz: oracle embeddings of ResNetArcFace([2,2,2,2], use_se=False) with the seeded weights of
``codeformer_b200.arcface.random_arcface_state_dict(seed=1)``, for the 32 inputs of ``inputs()``: the gray identity inputs of
the committed faces (tests/golden/faces.npz), then seeded N(0, 0.5) noise.  Only the embeddings are stored; the tests rebuild
the inputs with ``inputs()``.  CPU only:  python -m oracle.gen_golden_arcface"""
import os

import numpy as np
import torch

from codeformer_b200.arcface import random_arcface_state_dict
from oracle import arcface_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def inputs():
    """The 32 inputs of the golden: the gray identity inputs of the committed faces, then seeded noise."""
    faces = np.load(os.path.join(GOLDEN, 'faces.npz'))['faces']
    gray = AO.gray_resize_for_identity(AO.faces_to_input(faces))
    g = torch.Generator().manual_seed(7)
    noise = 0.5 * torch.randn((32 - gray.shape[0], 1, 128, 128), generator=g)
    return torch.cat([gray, noise]).contiguous()


def main():
    torch.set_grad_enabled(False)
    sd = random_arcface_state_dict(seed=1)
    x = inputs()
    emb = AO.arcface_forward(sd, x)
    np.savez_compressed(os.path.join(GOLDEN, 'arcface.npz'), emb=emb.numpy())
    print('arcface.npz', tuple(x.shape), tuple(emb.shape), float(emb.abs().max()))


if __name__ == '__main__':
    main()
