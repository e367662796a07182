"""Host planning of RealESRGANer.enhance_batch on the CPU: the grouping of tile_plan's rectangles into equal-shape forwards,
the composed reflect index map of pre_process, and the max_tiles chunking."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200.upsampler import reflect_pad_index, unshuffle_factor

# (height, width, scale, tile, tile_pad, pre_pad): sizes that are not multiples of the tile, an odd size at scale 2 (mod pad),
# scale 4, whole-image mode
CASES = [(75, 61, 2, 32, 8, 0), (75, 61, 2, 32, 8, 10), (64, 96, 2, 32, 8, 0), (37, 53, 4, 16, 4, 0), (37, 53, 4, 16, 4, 10),
         (41, 30, 1, 16, 4, 10), (33, 47, 2, 0, 10, 10), (512, 512, 2, 400, 40, 0), (1080, 1920, 2, 400, 40, 0)]


class Nearest(torch.nn.Module):
    """A stand-in model whose output pixel (y, x) is input pixel (y // scale, x // scale)."""

    def __init__(self, scale):
        super().__init__()
        self.scale = scale

    def forward(self, x):
        return x.repeat_interleave(self.scale, 2).repeat_interleave(self.scale, 3)


def _upsampler(scale, tile, tile_pad, pre_pad):
    return cb.RealESRGANer(scale=scale, model=Nearest(scale), tile=tile, tile_pad=tile_pad, pre_pad=pre_pad, device='cpu')


def _apply(er, groups, imgs):
    """What the uint8 tile forward does with the plan, with the stand-in model: read each window of the padded image
    through the index map, run the model, write the crop into the canvas where it falls inside.  Also counts the writes."""
    B, H, W, _ = imgs.shape
    s = er.scale
    padded = imgs[:, reflect_pad_index(H, er.pre_pad, s)][:, :, reflect_pad_index(W, er.pre_pad, s)]
    out = np.zeros((B, H * s, W * s, 3), imgs.dtype)
    hits = np.zeros((B, H * s, W * s), np.int64)
    for th, tw, rows in groups:
        for b, iy, ix, cy, cx, ch, cw, oy, ox in rows:
            win = padded[b, iy:iy + th, ix:ix + tw]
            assert win.shape[:2] == (th, tw), 'window outside the padded image'
            assert 0 <= cy and cy + ch <= th * s and 0 <= cx and cx + cw <= tw * s
            up = win.repeat(s, 0).repeat(s, 1)[cy:cy + ch, cx:cx + cw]
            y1, x1 = min(oy + ch, H * s), min(ox + cw, W * s)
            out[b, oy:y1, ox:x1] = up[:y1 - oy, :x1 - ox]
            hits[b, oy:y1, ox:x1] += 1
    return out, hits


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_groups_cover_every_output_pixel_once_and_match_the_tile_loop(case):
    H, W, s, tile, pad, pre = case
    er = _upsampler(s, tile, pad, pre)
    imgs = np.random.default_rng(H * W).random((2, H, W, 3), dtype=np.float32)
    groups = er.tile_groups(2, H, W, max_tiles=10 ** 6)
    assert len({(th, tw) for th, tw, _ in groups}) == len(groups), 'one forward per window shape without a limit'
    out, hits = _apply(er, groups, imgs)
    assert (hits == 1).all()
    if H * W <= 1 << 16:          # the reference chain on the stand-in model
        for b in range(2):
            ref = er._run(imgs[b][:, :, ::-1])          # _run takes RGB and returns BGR
            assert np.array_equal(out[b], ref)


def _mod_pad(n, pre, scale):
    m = unshuffle_factor(scale)
    return (m - (n + pre) % m) % m


# sizes where F.pad reflect accepts both pads: each smaller than the dimension it reflects
PAD_CASES = [(n, pre, scale) for n in (1, 2, 5, 6, 7, 37, 64) for pre in (0, 1, 4, 10) for scale in (1, 2, 4)
             if pre < n and _mod_pad(n, pre, scale) < n + pre]


@pytest.mark.parametrize('n,pre,scale', PAD_CASES)
def test_reflect_index_map_equals_two_reflect_pads(n, pre, scale):
    mod = _mod_pad(n, pre, scale)
    idx = np.arange(n)[:, None] * 1000 + np.arange(n)[None, :]          # an index image: row * 1000 + column
    x = torch.from_numpy(idx).double().view(1, 1, n, n)
    ref = F.pad(F.pad(x, (0, pre, 0, pre), 'reflect'), (0, mod, 0, mod), 'reflect')[0, 0].long().numpy()
    r = reflect_pad_index(n, pre, scale)
    assert np.array_equal(idx[r][:, r], ref)


def test_max_tiles_chunking_is_a_pure_function_of_the_sizes():
    er = _upsampler(2, 400, 40, 0)
    full = er.tile_groups(8, 1080, 1920, max_tiles=10 ** 6)
    assert len(full) == 9 and sum(len(r) for _, _, r in full) == 8 * 15
    for k in (1, 3, 7):
        g = er.tile_groups(8, 1080, 1920, max_tiles=k)
        assert g == er.tile_groups(8, 1080, 1920, max_tiles=k)
        assert all(1 <= len(r) <= k for _, _, r in g)
        # chunking only cuts each shape's list of tiles, in order
        for th, tw, rows in full:
            assert [t for h, w, r in g if (h, w) == (th, tw) for t in r] == rows


def test_default_chunks_keep_the_workspace_budget():
    net = cb.RRDBNet(3, 3, scale=2, num_block=1)
    lib = cb._lib.load()

    def tile_bytes(n, th, tw):
        return lib.cfb_rrdb_workspace_bytes(net._handle(), n, th, tw)
    er = cb.RealESRGANer(scale=2, model=Nearest(2), tile=400, tile_pad=40, pre_pad=0, device='cpu')
    groups = er.tile_groups(8, 1080, 1920, tile_bytes=tile_bytes)
    assert groups == er.tile_groups(8, 1080, 1920, tile_bytes=tile_bytes)
    budget = er.WORKSPACE_BUDGET
    for th, tw, rows in groups:
        assert tile_bytes(len(rows), th, tw) <= budget
    per_shape = {}
    for th, tw, rows in groups:
        per_shape.setdefault((th, tw), []).append(len(rows))
    for (th, tw), sizes in per_shape.items():       # every chunk but the last is full: one more tile would not fit
        assert tile_bytes(sizes[0] + 1, th, tw) > budget or len(sizes) == 1
    assert max(per_shape[(480, 480)]) == 6          # 0.69 GB per 480 x 480 tile at x2, 4 GiB budget
    big = cb.RealESRGANer(scale=2, model=Nearest(2), tile=0, pre_pad=0, device='cpu')
    assert [len(r) for _, _, r in big.tile_groups(2, 4000, 4000, tile_bytes=tile_bytes)] == [1, 1], 'at least one tile'
