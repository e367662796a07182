"""Write tests/golden/codeformer_fp16.npz: what CodeFormer / VQAutoEncoder in fp16 mode are compared against on the GPU.

The float64 emulation of the fp16 mode (tests/codeformer_fp16_emul.py) is run on the CPU on the cases of the reference golden
vectors, and stored are
  <case>_err   max-abs of the emulated `out` against the reference's fp32 output (the golden of that case, same sampling);
  u8_face0     the restored uint8 BGR face of face 0 (w=0.5, adain) through the caller's plumbing, emulated.
Cases: main (codeformer_main.npz: face 0, w=0.5, adain), w0 (codeformer_variants.npz: face 1, w=0, adain), c3 (face 1,
connect_list 32/64/128, w=0.7, adain) and vqae (vqae.npz: face 0).  The emulated code indices must equal the golden ones.

    python tools/gen_codeformer_fp16_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from codeformer_b200 import spec as S                    # noqa: E402
from oracle import plumbing_oracle as P                  # noqa: E402
from tests import codeformer_fp16_emul as CE             # noqa: E402
from tests.util import GOLDEN, faces_input, golden, maxabs   # noqa: E402

C3 = ('32', '64', '128')


def cases():
    """-> {name: (emulated out as the golden samples it, golden out, emulated indices, golden indices)}"""
    main, var, vq = golden('codeformer_main.npz'), golden('codeformer_variants.npz'), golden('vqae.npz')
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    res = {}
    o, _, _, idx = CE.codeformer_forward(sd, faces_input(slice(0, 1)), w=0.5, adain_on=True)
    res['main'] = (o, main['out'], idx[..., 0].numpy(), main['top_idx'])
    o, _, _, idx = CE.codeformer_forward(sd, faces_input(slice(1, 2)), w=0.0, adain_on=True)
    res['w0'] = (o[..., ::4, ::4], var['w0_out'], idx[..., 0].numpy(), var['w0_idx'])
    sd3 = S.random_state_dict(S.codeformer_spec(connect_list=C3), 3)
    o, _, _, idx = CE.codeformer_forward(sd3, faces_input(slice(1, 2)), w=0.7, adain_on=True, connect_list=C3)
    res['c3'] = (o[..., ::4, ::4], var['c3_out'], idx[..., 0].numpy(), var['c3_idx'])
    o, idx = CE.vqae_forward(S.random_state_dict(S.vqae_spec(), 2), faces_input(slice(0, 1)))
    res['vqae'] = (o[..., ::4, ::4], vq['out'], idx.numpy(), vq['idx'])
    return res


def u8_face0():
    """restore_faces([face 0 as BGR], w=0.5, adain=True) in fp16 mode, emulated: plumbing in, forward, plumbing out."""
    bgr = np.ascontiguousarray(golden('faces.npz')['faces'][:1][..., ::-1])
    x = torch.from_numpy(P.face_to_input(bgr))
    o = CE.codeformer_forward(S.random_state_dict(S.codeformer_spec(), 1), x, w=0.5, adain_on=True)[0]
    return P.output_to_face(o.float().numpy())


def main():
    torch.set_grad_enabled(False)
    out = {}
    for name, (emul, ref, idx, ref_idx) in cases().items():
        assert np.array_equal(idx.reshape(ref_idx.shape), ref_idx), f'{name}: emulated code indices differ from the golden'
        out[name + '_err'] = np.float64(maxabs(emul, ref))
        print(f'{name}: emulated out vs reference golden max-abs {float(out[name + "_err"]):.4e} '
              f'(|out|max {float(np.abs(ref).max()):.2f})')
    out['u8_face0'] = u8_face0()
    path = os.path.join(GOLDEN, 'codeformer_fp16.npz')
    np.savez_compressed(path, **out)
    print('wrote', path)


if __name__ == '__main__':
    main()
