"""A/B of two builds of libcfb200.so on the 128-wide halo tiles: a reference build (loaded through CFB_LIB) against the in-tree build.

Every measurement runs in a process of its own per build, alternating reference / in-tree for --rounds rounds, and reports the
median and range per build.  The card name and power limit are read in the same run.
  bench    bench.py --steps 10 --no-extras --no-cpu-baseline: `value` (faces/s)
  shapes   at batch 32, CUDA events around --reps launches: the 128-wide shapes of tools/conv_tile_sweep.py
           (cfb_debug_time_conv) and GN+SiLU conv 128->128 @256^2 with GroupNorm partials and the epilogues of the forward
           (residual, SFT + operand planes, both), in fp32 (split) and fp16 (single-pass) precision (cfb_debug_conv_tc_prec)
  outputs  bench.py --dump-outputs of both builds, and CodeFormer.forward in fp16 precision on bench.py's inputs: equal bit for bit

    python tools/wide_tile_ab.py --ref build/parent/libcfb200.so [--rounds 3] [--what bench,shapes,outputs]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from conv_tile_sweep import CHILD as SWEEP_CHILD, SHAPES, gpu_info      # noqa: E402

WIDE = [s for s in SHAPES if s[2] % 128 == 0]
# (residual, SFT, operand planes) of GN+SiLU conv 128->128 @256^2, all with GroupNorm partials (CPG 4)
EPILOGUES = [(False, False, False), (True, False, False), (False, True, True), (True, True, True)]

EPI_CHILD = r'''
import ctypes, json, sys
import torch
sys.path.insert(0, %r)
from codeformer_b200 import _lib
lib = _lib.load()
N, reps = int(sys.argv[1]), int(sys.argv[2])
H, C = 256, 128
g = torch.Generator().manual_seed(5)
x = torch.randn(N, H, H, C, generator=g).cuda()
w = (torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5).cuda()
b = (0.1 * torch.randn(C, generator=g)).cuda()
sc = (1 + 0.1 * torch.randn(N, C, generator=g)).cuda()
sh = (0.1 * torch.randn(N, C, generator=g)).cuda()
r = torch.randn(N, H, H, C, generator=g).cuda()
dec = torch.randn(N, H, H, C, generator=g).cuda()
scl = (0.5 * torch.randn(N, H, H, C, generator=g)).cuda()
out = torch.empty(N, H, H, C, device='cuda')
plane = (N * H * H * C * 2 + 1023) // 1024 * 1024
pl = torch.empty(2 * plane, dtype=torch.uint8, device='cuda')
gp = torch.empty(N * H * H // 128 * 4 * 64, device='cuda')
wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, C, C, 3, 0)
ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
tn = ctypes.c_int32(0)
res = []
for precision in (0, 1):
    for resid, sft, planes in json.loads(sys.argv[3]):
        def call():
            _lib.check(lib.cfb_debug_conv_tc_prec(
                _lib.ptr(x), None, 0, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), N, H, H, C, C, 0, 1, _lib.ptr(sc), _lib.ptr(sh), 1,
                _lib.ptr(r) if resid else None, _lib.ptr(dec) if sft else None, _lib.ptr(scl) if sft else None, 0.5,
                _lib.ptr(pl) if planes else None, _lib.ptr(gp), _lib.ptr(ws), wsb, st, ctypes.byref(tn), 3, 0, precision),
                'cfb_debug_conv_tc_prec')
        for _ in range(2):
            call()
        torch.cuda.synchronize()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call()
        e.record()
        e.synchronize()
        assert tn.value == 128, tn.value
        res.append(a.elapsed_time(e) / reps)
print('RESULT ' + json.dumps(res))
''' % ROOT

FP16_CHILD = r'''
import sys
import numpy as np
import torch
sys.path.insert(0, %r)
import codeformer_b200 as cb
from codeformer_b200 import spec as S
torch.set_grad_enabled(False)
net = cb.CodeFormer(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                    connect_list=['32', '64', '128', '256']).cuda().eval()
net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
net.set_precision('fp16')
g = torch.Generator().manual_seed(100)
x = torch.randn(32, 3, 512, 512, generator=g).clamp_(-1, 1).cuda()
out, logits, lq = net(x, w=0.5, adain=True)
torch.cuda.synchronize()
np.savez(sys.argv[1], out=out.cpu().numpy(), logits=logits.cpu().numpy(), lq_feat=lq.cpu().numpy())
print('RESULT saved')
''' % ROOT


def run(cmd, lib, timeout=3600):
    env = dict(os.environ)
    env.pop('CFB_LIB', None)
    if lib:
        env['CFB_LIB'] = lib
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError(' '.join(cmd[:3]) + '\n' + p.stdout[-3000:] + p.stderr[-3000:])
    return p.stdout


def result(stdout):
    return json.loads([ln for ln in stdout.splitlines() if ln.startswith('RESULT ')][-1][len('RESULT '):])


def bench_value(stdout):
    return [json.loads(ln) for ln in stdout.splitlines() if ln.startswith('{')][-1]['value']


def summary(xs):
    return {'median': round(statistics.median(xs), 4), 'min': round(min(xs), 4), 'max': round(max(xs), 4), 'runs': [round(v, 4) for v in xs]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--ref', required=True, help='reference libcfb200.so (CFB_LIB)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--what', default='outputs,bench,shapes')
    args = ap.parse_args()
    ref = os.path.abspath(args.ref)
    what = args.what.split(',')
    sides = (('ref', ref), ('new', None))
    print(json.dumps({'gpu': gpu_info(), 'ref': os.path.relpath(ref, ROOT), 'rounds': args.rounds}), flush=True)
    if 'outputs' in what:
        import numpy as np
        tmp = tempfile.mkdtemp(prefix='wide_tile_ab_')
        for name, lib in sides:
            run([sys.executable, 'bench.py', '--steps', '2', '--warmup', '1', '--no-extras', '--no-cpu-baseline',
                 '--dump-outputs', os.path.join(tmp, name)], lib)
            run([sys.executable, '-c', FP16_CHILD, os.path.join(tmp, name + '_fp16.npz')], lib)
        same = {}
        for f in sorted(os.listdir(os.path.join(tmp, 'ref'))):
            a, b = np.load(os.path.join(tmp, 'ref', f)), np.load(os.path.join(tmp, 'new', f))
            same['fp32 ' + f] = bool(a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)))
        a, b = np.load(os.path.join(tmp, 'ref_fp16.npz')), np.load(os.path.join(tmp, 'new_fp16.npz'))
        for k in a.files:
            same['fp16 ' + k] = bool(np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)))
        print(json.dumps({'bit_identical': same}), flush=True)
    if 'bench' in what:
        vals = {'ref': [], 'new': []}
        for _ in range(args.rounds):
            for name, lib in sides:
                vals[name].append(bench_value(run([sys.executable, 'bench.py', '--gpus', '1', '--steps', '10',
                                                   '--no-extras', '--no-cpu-baseline'], lib)))
        print(json.dumps({'bench_value_faces_per_s': {k: summary(v) for k, v in vals.items()}}), flush=True)
    if 'shapes' in what:
        t = {'ref': [], 'new': []}
        for _ in range(args.rounds):
            for name, lib in sides:
                sw = result(run([sys.executable, '-c', SWEEP_CHILD, str(args.batch), str(args.reps), json.dumps(WIDE)], lib))
                ep = result(run([sys.executable, '-c', EPI_CHILD, str(args.batch), str(args.reps), json.dumps(EPILOGUES)], lib))
                t[name].append(sw + ep)
        labels = [f'{"up" if m == 2 else "conv"} {ci}->{co} @{2 * h if m == 2 else h}^2{" gn+silu" if xf else " raw"}'
                  for h, ci, co, m, xf in WIDE]
        labels += [f'{prec} gn+silu 128->128 @256^2 gn' + ('+res' if r else '') + ('+sft' if s else '') + ('+planes' if p else '')
                   for prec in ('fp32', 'fp16') for r, s, p in EPILOGUES]
        for i, lab in enumerate(labels):
            ref_ms, new_ms = summary([v[i] for v in t['ref']]), summary([v[i] for v in t['new']])
            print(json.dumps({'shape': lab, 'ref_ms': ref_ms['median'], 'ref_range': [ref_ms['min'], ref_ms['max']],
                              'new_ms': new_ms['median'], 'new_range': [new_ms['min'], new_ms['max']],
                              'speedup': round(ref_ms['median'] / new_ms['median'], 3)}), flush=True)


if __name__ == '__main__':
    main()
