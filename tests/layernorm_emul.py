"""Float32 restatement of the LayerNorm kernel (simt_kernels.cu: layer_norm_kernel), the token-row classes it is tested on and
the float64 bar the GPU test (tests/test_gpu_transformer_stage.py) holds both of its forms to.

The kernel normalises one row of C = 512 values per warp: lane l holds the float4s at channels (i * 32 + l) * 4, i < 4, and
adds each as (x + y) + (z + w) to its running sum; an xor butterfly over the 32 lanes gives every lane the row sum, the mean
is sum / C.  The variance is a second pass over the deviations from that mean (the same lane order), rstd = rsqrtf(sq / C +
1e-5), y = (x - mean) * rstd * gamma + beta.  numpy float32 rounds every operation to nearest like the kernel (which may
contract some products into FMAs; rsqrtf is within 2 ulp): the restatement reproduces the kernel's error model, not its bits.

Errors are measured per element in units of |gamma_c| (the normalised value has unit spread): with r = |row mean| / row
standard deviation the fp32 arithmetic errs like r * 2^-24 -- the rounding of x - mean, which no fp32 kernel avoids, and of
the mean itself.  The bar is LN_K x the error of float32 torch (F.layer_norm on the CPU) against float64 + LN_FLOOR, per row
class."""
import numpy as np
import torch
import torch.nn.functional as F

F32 = np.float32
C = 512
EPS = 1e-5
LANES, V = 32, C // 128

# The bar: the kernel's mean is a tree sum where torch's CPU kernel sums in another order, so their mean errors differ by a
# small factor (the restatement below: at most 1.3x torch's error over the row classes); 4x leaves room for the FMA
# contractions and rsqrtf.  The floor covers rows where torch is exact (constant rows: y = beta) and a few fp32 ulps of |y|
# elsewhere (|y| / |gamma| < 25 on these rows).
LN_K = 4.0
LN_FLOOR = 2e-6

# r = |mean| / std of the DC-offset classes
R_VALUES = (1e2, 1e3, 1e4)


def row_classes(T, seed):
    """-> (x [T, C] fp32, {class name: row indices}): T rows in eight classes, assigned round-robin (so every class has rows
    of every image and every position of a 256-token image when T = 3 * 256): benign N(0.3, 2); DC offsets of r standard
    deviations (sign alternating per row); one massive channel (1e3 x the others); near-constant rows (std 1e-4 < sqrt(eps)
    around 0.5); exactly constant rows (2.0, exact in binary, and 0.1, not exact)."""
    g = np.random.default_rng(seed)
    z = g.standard_normal((T, C))
    names = ['benign'] + [f'dc r={r:g}' for r in R_VALUES] + ['massive channel', 'near-constant', 'constant 2', 'constant 0.1']
    cls = np.arange(T) % len(names)
    x = 0.3 + 2.0 * z
    sign = np.where((np.arange(T) // len(names)) % 2 == 0, 1.0, -1.0)[:, None]
    for i, r in enumerate(R_VALUES):
        m = cls == 1 + i
        x[m] = sign[m] * r * 1.5 + 1.5 * z[m]
    m = cls == 4
    ch = g.integers(0, C, size=T)
    x[m, ch[m]] = 1e3 * np.sign(z[m, ch[m]] + 1e-30) * (1 + np.abs(z[m, ch[m]]))
    x[cls == 5] = 0.5 + 1e-4 * z[cls == 5]
    x[cls == 6] = 2.0
    x[cls == 7] = 0.1
    return x.astype(F32), {n: np.nonzero(cls == i)[0] for i, n in enumerate(names)}


def affine(seed):
    """nontrivial gamma (|gamma| in [0.25, 3], both signs) and beta"""
    g = np.random.default_rng(seed)
    gamma = np.where(g.random(C) < 0.3, -1.0, 1.0) * (0.25 + np.abs(g.standard_normal(C)))
    gamma = np.clip(gamma, -3, 3)
    return gamma.astype(F32), (0.5 * g.standard_normal(C)).astype(F32)


def _lanes(x):
    """[T, C] -> [T, V, LANES, 4]: element [t, i, l, k] is channel (i * 32 + l) * 4 + k"""
    return x.reshape(x.shape[0], V, LANES, 4)


def _butterfly(s):
    """xor butterfly over the lane axis (last): every lane ends with the same row total"""
    lane = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s


def _lane_sum(q):
    """per-lane running sum over i of (a + b) + (c + d), q [T, V, LANES, 4] -> [T, LANES]"""
    s = np.zeros((q.shape[0], LANES), F32)
    for i in range(V):
        s = s + ((q[:, i, :, 0] + q[:, i, :, 1]) + (q[:, i, :, 2] + q[:, i, :, 3]))
    return s


def layer_norm_f32(x, gamma, beta, mutant=None):
    """The kernel's arithmetic in float32; ``mutant``: 'one_pass' (var = E[x^2] - mean^2), 'eps' (1e-6), 'drop_float4' (the
    mean misses lane 0's last float4, as a lane partition with one float4 too few would)."""
    x = x.astype(F32)
    q = _lanes(x)
    inv_c = F32(1.0 / C)
    if mutant == 'drop_float4':
        qm = q.copy()
        qm[:, V - 1, 0, :] = 0
        mean = _butterfly(_lane_sum(qm))[:, :1] * inv_c
    else:
        mean = _butterfly(_lane_sum(q))[:, :1] * inv_c
    if mutant == 'one_pass':
        var = _butterfly(_lane_sum(q * q))[:, :1] * inv_c - mean * mean
        var = np.maximum(var, F32(0))
    else:
        d = q - mean[:, :, None, None]
        var = _butterfly(_lane_sum(d * d))[:, :1] * inv_c
    eps = F32(1e-6 if mutant == 'eps' else EPS)
    rstd = (1.0 / np.sqrt((var + eps).astype(np.float64))).astype(F32)
    return ((x - mean) * rstd) * gamma + beta


def reference(x, gamma, beta):
    """float64 F.layer_norm of the fp32 input, and float32 torch's own result"""
    xt, gt, bt = (torch.from_numpy(np.asarray(a)) for a in (x, gamma, beta))
    y64 = F.layer_norm(xt.double(), (C,), gt.double(), bt.double(), eps=EPS).numpy()
    y32 = F.layer_norm(xt, (C,), gt, bt, eps=EPS).numpy()
    return y64, y32


def unit_errors(y, y64, gamma):
    """|y - y64| / |gamma_c| per element (NaN counts as infinite)"""
    e = np.abs(np.asarray(y, np.float64) - y64) / np.abs(gamma.astype(np.float64))
    return np.where(np.isnan(e), np.inf, e)


def judge(what, err, e32, failures, k=LN_K, floor=LN_FLOOR):
    """one line per case: kernel error, float32 torch's error, the bar; a failure is appended to ``failures``"""
    bar = k * e32 + floor
    print(f'{what:44s} kernel {err:.3e}  torch32 {e32:.3e}  bar {bar:.3e}' + ('' if err <= bar else '  FAIL'))
    if not err <= bar:
        failures.append(f'{what}: {err:.3e} > {k:g} x {e32:.3e} + {floor:g}')


def class_errors(y, y64, y32, gamma, classes):
    """{class: (max error of y, max error of float32 torch)} in units of |gamma|"""
    ek, et = unit_errors(y, y64, gamma), unit_errors(y32, y64, gamma)
    return {n: (float(ek[rows].max()), float(et[rows].max())) for n, rows in classes.items()}
