"""CPU model of the GroupNorm partial slots (kernels.cuh: gn_lane_moments / gn_merge_xor, simt_kernels.cu: gn_final_f32_kernel,
gn_cat_partials_kernel): why a slot holds (mean, M2) rather than (sum, sum of squares).

A slot covers 32 pixels x 4 channels of one group, as in the 128-wide conv epilogue: four lanes with 8 rows x 4 channels each,
summed in fp32, merged pairwise over the lanes, then all slots of the image finalized in float64.  With r = |group mean| /
group standard deviation, the relative error of rstd against float64 grows like
  * (1 + r^2) * 2^-24 for fp32 (sum, sum of squares): the variance cancels against mean^2;
  * r * 2^-24 for (mean, M2) around a per-lane shift: only the rounding of the slot means is left.
No GPU involved; numpy float32 rounds every operation to nearest like the kernels (which contract some products into FMAs)."""
import numpy as np

F32 = np.float32
U = 2.0 ** -24
EPS = 1e-6


def group(r, seed, pixels=4096, cpg=4):
    """one group's values as [slots, 4 lanes, 32 values] fp32: offset r, unit standard deviation, a per-channel spread"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((pixels, cpg)) * 0.9 + rng.standard_normal(cpg) * 0.4 + r
    return x.reshape(pixels // 32, 4, 8, cpg).reshape(pixels // 32, 4, 32).astype(F32)


def exact_rstd(x):
    v = x.astype(np.float64).reshape(-1)
    return 1.0 / np.sqrt(v.var() + EPS)


def rstd_power_sums(x):
    """the previous format: fp32 sum and sum of squares per lane, lane sums added pairwise, float64 finalize"""
    s = np.zeros(x.shape[:2], F32)
    q = np.zeros(x.shape[:2], F32)
    for i in range(x.shape[2]):
        s = s + x[..., i]
        q = q + x[..., i] * x[..., i]
    s, q = (s[:, 0] + s[:, 1]) + (s[:, 2] + s[:, 3]), (q[:, 0] + q[:, 1]) + (q[:, 2] + q[:, 3])
    n = x.size
    mean = s.astype(np.float64).sum() / n
    var = max(q.astype(np.float64).sum() / n - mean * mean, 0.0)
    return 1.0 / np.sqrt(var + EPS)


def lane_moments(x):
    """gn_lane_moments: sums of the deviations from the lane's first value -> (mean, M2) of the lane's values"""
    k = x[..., 0]
    s = np.zeros(x.shape[:-1], F32)
    q = np.zeros(x.shape[:-1], F32)
    for i in range(x.shape[-1]):
        d = x[..., i] - k
        s = s + d
        q = q + d * d
    dm = s * F32(1.0 / x.shape[-1])
    return k + dm, np.maximum(q - s * dm, F32(0))


def merge(ma, qa, mb, qb, n):
    """gn_merge_xor / gn_cat_partials_kernel: two (mean, M2) of n values each"""
    d = ma - mb
    return F32(0.5) * (ma + mb), (qa + qb) + (d * d) * F32(0.5 * n)


def slots_moments(x):
    m, q = lane_moments(x)
    n = x.shape[-1]
    m01, q01 = merge(m[:, 0], q[:, 0], m[:, 1], q[:, 1], n)
    m23, q23 = merge(m[:, 2], q[:, 2], m[:, 3], q[:, 3], n)
    return merge(m01, q01, m23, q23, 2 * n)


def finalize(mean, m2, per_slot):
    """gn_final_f32_kernel: float64 sums of the slots' deviations from slot 0's mean"""
    K = float(mean[0])
    d = mean.astype(np.float64) - K
    a, b = d.sum(), (m2.astype(np.float64) + per_slot * d * d).sum()
    S = mean.size
    var = max(b / (S * per_slot) - (a / S) ** 2, 0.0)
    return 1.0 / np.sqrt(var + EPS), K + a / S


def rel_errors(r, seeds=range(4)):
    old, new = [], []
    for s in seeds:
        x = group(r, s)
        ref = exact_rstd(x)
        old.append(abs(rstd_power_sums(x) / ref - 1))
        m, q = slots_moments(x)
        new.append(abs(finalize(m, q, 128)[0] / ref - 1))
    return max(old), max(new)


def test_moments_error_grows_like_r():
    for r in (0, 10, 100, 1000, 10000):
        _, new = rel_errors(r)
        assert new <= 8 * (1 + r) * U, (r, new)


def test_power_sums_error_grows_like_r_squared():
    old100, new100 = rel_errors(100)
    old1000, new1000 = rel_errors(1000)
    assert old100 > 10 * new100 and old1000 > 100 * new1000
    assert old1000 > 30 * old100                   # r x10 -> error x~100
    assert old1000 > 1e-3                          # percents of rstd lost at r = 1000: the reason for the format


def test_constant_and_tiny_groups_are_exact():
    """a constant group (exact or not in binary) gives M2 = 0 and its own value as the mean"""
    for v in (2.0, 0.1, -1234.567):
        x = np.full((128, 4, 32), v, F32)
        m, q = slots_moments(x)
        rstd, mean = finalize(m, q, 128)
        assert mean == float(F32(v)) and rstd == 1.0 / np.sqrt(EPS)
    rng = np.random.default_rng(9)
    x = (0.5 + 1e-4 * rng.standard_normal((128, 4, 32))).astype(F32)       # std 0.1 sqrt(eps): eps dominates
    m, q = slots_moments(x)
    assert abs(finalize(m, q, 128)[0] / exact_rstd(x) - 1) < 1e-6


def test_concatenation_merge():
    """gn_cat_partials: group g of cat([a, b]) from groups 2g, 2g+1 of one source, 128 values per slot each"""
    a, b = group(1000, 1), group(1000, 2)
    ma, qa = slots_moments(a)
    mb, qb = slots_moments(b)
    m, q = merge(ma, qa, mb, qb, 128)
    both = np.concatenate([a, b], axis=2)
    rstd, mean = finalize(m, q, 256)
    assert abs(rstd / exact_rstd(both) - 1) <= 8 * 1001 * U
    assert abs(mean - both.astype(np.float64).mean()) <= 4 * U * 1000
