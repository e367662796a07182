"""Where the 128 x 128 halo tiles wait: per-role wait counters of the GN+SiLU convs with the epilogues of the forward.

Builds the library with -DCFB_TC_STAMPS=1 into build/epilogue_waits/ (rebuilt when a source is newer) and runs, in a process
that loads that build (CFB_LIB), GN+SiLU conv 128->128 and 256->128 @256^2 at batch 32 with GroupNorm partials and each
epilogue of the forward (none, residual, SFT + operand planes, all three), in fp32 (split) and fp16 (single-pass) precision,
through cfb_debug_conv_tc_prec.  Every CTA adds the cycles its roles spend in each wait to its counters (conv_tc.cu, TC_CNT0);
printed are the shares of each role's cycles, summed over the CTAs and the timed launches:
  mma   weight `full` wait, patch `afull` wait, `cempty` wait before the tile hand-off (each over the MMA warps' role cycles)
  epi   `cfull` wait, residual / SFT loads (issue until the batch has arrived), stores (output, operand planes, GroupNorm
        partials) (each over the epilogue warps' role cycles)
and the kernel time of the stamps build (CUDA events; the counters slow it, so compare rows with each other, not with the
production build).  The card name and power limit are read in the same run.

    python tools/epilogue_waits.py [--batch 32] [--reps 5] [--lib DIR/libcfb200.so]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from conv_tile_sweep import gpu_info      # noqa: E402

OUT_DIR = os.path.join(ROOT, 'build', 'epilogue_waits')
# (residual, SFT, operand planes), all with GroupNorm partials
EPILOGUES = [(False, False, False), (True, False, False), (False, True, True), (True, True, True)]
SHAPES = [(256, 128, 128), (256, 256, 128)]          # (H, Cin, Cout), 3x3 'same', GroupNorm + SiLU input
NCNT, CNT0 = 8, 32                                   # conv_tc.cu: TC_NCNT, TC_CNT0

CHILD = r'''
import ctypes, json, sys
import torch
sys.path.insert(0, %r)
from codeformer_b200 import _lib
lib = _lib.load()
N, reps = int(sys.argv[1]), int(sys.argv[2])
shapes, epilogues = json.loads(sys.argv[3]), json.loads(sys.argv[4])
NCNT, CNT0 = %d, %d
sms = torch.cuda.get_device_properties(0).multi_processor_count
dbg = torch.zeros(CNT0 + NCNT * sms, dtype=torch.int64, device='cuda')
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
tn = ctypes.c_int32(0)
res = []
for H, Cin, C in shapes:
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, H, H, Cin, generator=g).cuda()
    w = (torch.randn(C, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).cuda()
    b = (0.1 * torch.randn(C, generator=g)).cuda()
    sc = (1 + 0.1 * torch.randn(N, Cin, generator=g)).cuda()
    sh = (0.1 * torch.randn(N, Cin, generator=g)).cuda()
    r = torch.randn(N, H, H, C, generator=g).cuda()
    dec = torch.randn(N, H, H, C, generator=g).cuda()
    scl = (0.5 * torch.randn(N, H, H, C, generator=g)).cuda()
    out = torch.empty(N, H, H, C, device='cuda')
    plane = (N * H * H * C * 2 + 1023) // 1024 * 1024
    pl = torch.empty(2 * plane, dtype=torch.uint8, device='cuda')
    gp = torch.empty(N * H * H // 128 * 4 * 64, device='cuda')
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, Cin, C, 3, 0)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    for precision in (0, 1):
        for resid, sft, planes in epilogues:
            def call():
                _lib.check(lib.cfb_debug_conv_tc_prec(
                    _lib.ptr(x), None, 0, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), N, H, H, Cin, C, 0, 1, _lib.ptr(sc),
                    _lib.ptr(sh), 1, _lib.ptr(r) if resid else None, _lib.ptr(dec) if sft else None,
                    _lib.ptr(scl) if sft else None, 0.5, _lib.ptr(pl) if planes else None, _lib.ptr(gp), _lib.ptr(ws), wsb,
                    st, ctypes.byref(tn), 3, 0, precision), 'cfb_debug_conv_tc_prec')
            for _ in range(2):
                call()
            torch.cuda.synchronize()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                call()
            e.record()
            e.synchronize()
            ms = a.elapsed_time(e) / reps
            dbg.zero_()
            _lib.check(lib.cfb_debug_set_stamps(_lib.ptr(dbg)), 'cfb_debug_set_stamps')
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
            _lib.check(lib.cfb_debug_set_stamps(None), 'cfb_debug_set_stamps')
            assert tn.value == 128, tn.value
            cnt = dbg[CNT0:].view(sms, NCNT).sum(0).tolist()
            res.append({'shape': [H, Cin, C], 'precision': precision, 'epilogue': [resid, sft, planes], 'ms': ms, 'cnt': cnt})
    del x, w, r, dec, scl, out, pl, gp, ws
    torch.cuda.empty_cache()
print('RESULT ' + json.dumps(res))
''' % (ROOT, NCNT, CNT0)


def build_stamps():
    """The stamps build of the library in OUT_DIR (build.py's staleness check decides whether to compile)."""
    lib = os.path.join(OUT_DIR, 'libcfb200.so')
    os.makedirs(OUT_DIR, exist_ok=True)
    env = dict(os.environ, CFB_BUILD_OUT=lib, CFB_NVCC_EXTRA='-DCFB_TC_STAMPS=1')
    env.pop('CFB_PTXAS_V', None)
    subprocess.run([sys.executable, '-c', 'from codeformer_b200 import build; build.build()'], cwd=ROOT, env=env, check=True,
                   stdout=subprocess.DEVNULL)
    return lib


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=5, help='timed launches per row (and launches counted)')
    ap.add_argument('--lib', help='an existing stamps build to use instead of building one')
    args = ap.parse_args()
    lib = os.path.abspath(args.lib) if args.lib else build_stamps()
    env = dict(os.environ, CFB_LIB=lib)
    p = subprocess.run([sys.executable, '-c', CHILD, str(args.batch), str(args.reps), json.dumps(SHAPES), json.dumps(EPILOGUES)],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=3600)
    if p.returncode != 0:
        raise RuntimeError(p.stdout[-3000:] + p.stderr[-3000:])
    rows = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')][-1][len('RESULT '):])
    print(json.dumps({'gpu': gpu_info(), 'batch': args.batch, 'reps': args.reps, 'lib': os.path.relpath(lib, ROOT)}))
    for r in rows:
        c = r['cnt']
        mma, epi = max(c[3], 1), max(c[7], 1)
        res, sft, planes = r['epilogue']
        H, Cin, C = r['shape']
        print(json.dumps({
            'shape': f'gn+silu {Cin}->{C} @{H}^2', 'precision': 'fp16' if r['precision'] else 'fp32',
            'epilogue': 'gn' + ('+res' if res else '') + ('+sft' if sft else '') + ('+planes' if planes else ''),
            'ms_stamps_build': round(r['ms'], 3),
            'mma': {'full': round(c[0] / mma, 4), 'afull': round(c[1] / mma, 4), 'cempty': round(c[2] / mma, 4)},
            'epi': {'cfull': round(c[4] / epi, 4), 'loads': round(c[5] / epi, 4), 'stores': round(c[6] / epi, 4)},
            'mcycles': {'mma_role': round(c[3] / 1e6, 1), 'epi_role': round(c[7] / 1e6, 1)}}), flush=True)


if __name__ == '__main__':
    main()
