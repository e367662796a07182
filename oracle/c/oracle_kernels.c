/* CPU restatement in plain C of the integer/index steps of the hot path and of the direct convolution,
 * with double-precision accumulation -- TEST INFRASTRUCTURE (checker only; never linked by the product).
 *
 *   vq_nearest_ref     VectorQuantizer.forward distance + argmin   /root/reference/basicsr/archs/vqgan_arch.py:38-44
 *   argmax_lookup_ref  softmax->topk(1)->one-hot@E                 codeformer_arch.py:257-259, vqgan_arch.py:72-84
 *   conv2d_nhwc_ref    nn.Conv2d 3x3/1x1 (+Downsample/Upsample)    vqgan_arch.py:117-138,147-151
 *   group_norm_ref     GroupNorm(32,C,eps)                         vqgan_arch.py:14-15
 * "parity unpinned" by the reference (it ships no vectors); pinned by tests/golden (oracle/gen_golden.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* z [T,D], E [K,D] -> idx [T] = first index of the minimum of |z|^2+|e|^2-2 z.e (evaluated in double) */
void vq_nearest_ref(const float* z, const float* E, int T, int D, int K, int64_t* idx, double* min_gap) {
  double gap = INFINITY;
  for (int t = 0; t < T; ++t) {
    double best = INFINITY, second = INFINITY;
    int bi = 0;
    double z2 = 0;
    for (int d = 0; d < D; ++d) z2 += (double)z[(size_t)t * D + d] * z[(size_t)t * D + d];
    for (int k = 0; k < K; ++k) {
      double e2 = 0, ze = 0;
      for (int d = 0; d < D; ++d) {
        const double e = E[(size_t)k * D + d];
        e2 += e * e;
        ze += e * (double)z[(size_t)t * D + d];
      }
      const double dist = z2 + e2 - 2 * ze;
      if (dist < best) { second = best; best = dist; bi = k; }
      else if (dist < second) second = dist;
    }
    idx[t] = bi;
    if (second - best < gap) gap = second - best;
  }
  if (min_gap) *min_gap = gap;
}

/* logits [T,K] -> idx (first maximum), quant [T,D] = E[idx] */
void argmax_lookup_ref(const float* logits, const float* E, int T, int K, int D, int64_t* idx, float* quant) {
  for (int t = 0; t < T; ++t) {
    int bi = 0;
    float best = logits[(size_t)t * K];
    for (int k = 1; k < K; ++k)
      if (logits[(size_t)t * K + k] > best) { best = logits[(size_t)t * K + k]; bi = k; }
    idx[t] = bi;
    for (int d = 0; d < D; ++d) quant[(size_t)t * D + d] = E[(size_t)bi * D + d];
  }
}

/* in [N,H,W,Cin] NHWC, w OIHW [Cout,Cin,k,k], out [N,Ho,Wo,Cout]; mode 0 same, 1 down (pad r/b, s2), 2 up (nearest x2) */
void conv2d_nhwc_ref(const float* in, const float* w, const float* bias, float* out, int N, int H, int W, int Cin,
                     int Cout, int k, int mode) {
  const int Ho = mode == 1 ? H / 2 : (mode == 2 ? H * 2 : H), Wo = mode == 1 ? W / 2 : (mode == 2 ? W * 2 : W);
  for (int n = 0; n < N; ++n)
    for (int oy = 0; oy < Ho; ++oy)
      for (int ox = 0; ox < Wo; ++ox)
        for (int co = 0; co < Cout; ++co) {
          double acc = bias ? bias[co] : 0.0;
          for (int r = 0; r < k; ++r)
            for (int s = 0; s < k; ++s) {
              int iy, ix;
              if (mode == 1) { iy = oy * 2 + r; ix = ox * 2 + s; if (iy >= H || ix >= W) continue; }
              else if (mode == 2) {
                iy = oy + r - 1; ix = ox + s - 1;
                if (iy < 0 || ix < 0 || iy >= 2 * H || ix >= 2 * W) continue;
                iy >>= 1; ix >>= 1;
              } else {
                iy = oy + r - k / 2; ix = ox + s - k / 2;
                if (iy < 0 || ix < 0 || iy >= H || ix >= W) continue;
              }
              const float* ip = in + (((size_t)n * H + iy) * W + ix) * Cin;
              for (int ci = 0; ci < Cin; ++ci) acc += (double)ip[ci] * w[(((size_t)co * Cin + ci) * k + r) * k + s];
            }
          out[(((size_t)n * Ho + oy) * Wo + ox) * Cout + co] = (float)acc;
        }
}

/* x [N,HW,C] NHWC -> y = (x-mean_g)*rstd_g*gamma+beta, biased variance per (n, group) */
void group_norm_ref(const float* x, const float* gamma, const float* beta, float* y, int N, int HW, int C, int groups,
                    double eps) {
  const int cpg = C / groups;
  for (int n = 0; n < N; ++n)
    for (int g = 0; g < groups; ++g) {
      double s = 0, q = 0;
      for (int p = 0; p < HW; ++p)
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { const double v = x[((size_t)n * HW + p) * C + c]; s += v; q += v * v; }
      const double cnt = (double)HW * cpg, mean = s / cnt, var = q / cnt - mean * mean, rstd = 1.0 / sqrt(var + eps);
      for (int p = 0; p < HW; ++p)
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
          const size_t i = ((size_t)n * HW + p) * C + c;
          y[i] = (float)(((double)x[i] - mean) * rstd * gamma[c] + beta[c]);
        }
    }
}

/* ---- cv2 4.13's separable filters and float64 resize, as the paste-back calls them ---------------------------------
 * cv2.GaussianBlur(src, (n, n), sigma) on CV_32F / CV_64F is sepFilter2D with BORDER_REFLECT_101: a row pass into a
 * buffer of src's type, then a column pass.  Which arithmetic an output gets depends on the SIMD block it falls in, so
 * these restate cv2 4.13 as built for x86-64 with its AVX2 dispatch (the PyPI wheels); cv2's fused multiply-adds are fmaf /
 * fma here, and this file is built with -ffp-contract=off so that nothing else is fused.  k is the whole kernel (n taps).
 *
 *   float32 rows, n >= 7   x < w - w % 4: fmaf chain in tap order from 0.  The last w % 4 outputs: k[0] s[0], then taps
 *                          1 .. n - 1 in order, the first 4 * ((n - 1) / 4) added as rounded products, the rest fmaf'd.
 *   float32 rows, n == 5   x < w - w % 2: fmaf(s[0], k[2], p1 k[3]) + p2 k[4]; the last output of an odd width:
 *                          (s[0] k[2] + p1 k[3]) + p2 k[4], every step rounded.  p_i = s[+i] + s[-i], rounded.
 *   float32 rows, n == 3   s[0] k[1] + p1 k[2].
 *   float32 columns        x < w - w % 8: the centre product, then fmaf(p_i, k[r + i], acc) for i = 1 .. r.  The last
 *                          w % 8 columns: the same with rounded products and sums.  (n = 3 and 5 have dyadic kernels whose
 *                          products are exact, so their own small-kernel code agrees with this.)
 *   float64 rows           x < w - w % 4: fma chain in tap order from 0; the last w % 4 outputs: products and sums rounded.
 *   float64 columns        the centre product, then acc + p_i k[r + i] with every step rounded, for every column.
 * n == 1 copies.  tmp holds h * w values of the row pass. */
static int reflect101(int p, int n) {
  if (n == 1) return 0;
  const int per = 2 * (n - 1);
  int q = p % per;
  if (q < 0) q += per;
  return q >= n ? per - q : q;
}

static void blur_rows_f32(const float* src, float* dst, int h, int w, const float* k, int n) {
  const int r = n / 2, nvec = w - w % 4, nunf = 4 * ((n - 1) / 4);
#pragma omp parallel for
  for (int y = 0; y < h; ++y) {
    const float* s = src + (size_t)y * w;
    for (int x = 0; x < w; ++x) {
#define S(i) s[reflect101(x + (i), w)]
      float acc;
      if (n == 3) {
        acc = S(0) * k[1] + (S(-1) + S(1)) * k[2];
      } else if (n == 5) {
        const float p1 = S(-1) + S(1), p2 = S(-2) + S(2);
        if (x < w - w % 2) acc = fmaf(S(0), k[2], p1 * k[3]) + p2 * k[4];
        else { acc = S(0) * k[2] + p1 * k[3]; acc = acc + p2 * k[4]; }
      } else if (x < nvec) {
        acc = 0.f;
        for (int t = 0; t < n; ++t) acc = fmaf(S(t - r), k[t], acc);
      } else {
        acc = S(-r) * k[0];
        for (int t = 1; t < n; ++t) acc = t <= nunf ? acc + S(t - r) * k[t] : fmaf(S(t - r), k[t], acc);
      }
#undef S
      dst[(size_t)y * w + x] = acc;
    }
  }
}

static void blur_cols_f32(const float* src, float* dst, int h, int w, const float* k, int n) {
  const int r = n / 2, nvec = w - w % 8;
#pragma omp parallel for
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float acc = src[(size_t)y * w + x] * k[r];
      for (int i = 1; i <= r; ++i) {
        const float p = src[(size_t)reflect101(y + i, h) * w + x] + src[(size_t)reflect101(y - i, h) * w + x];
        acc = x < nvec ? fmaf(p, k[r + i], acc) : acc + p * k[r + i];
      }
      dst[(size_t)y * w + x] = acc;
    }
}

void gauss_blur_f32_ref(const float* src, float* dst, float* tmp, int h, int w, const float* k, int n) {
  if (n == 1) { memcpy(dst, src, (size_t)h * w * sizeof(float)); return; }
  blur_rows_f32(src, tmp, h, w, k, n);
  blur_cols_f32(tmp, dst, h, w, k, n);
}

void gauss_blur_f64_ref(const double* src, double* dst, double* tmp, int h, int w, const double* k, int n) {
  const int r = n / 2, nvec = w - w % 4;
#pragma omp parallel for
  for (int y = 0; y < h; ++y) {
    const double* s = src + (size_t)y * w;
    for (int x = 0; x < w; ++x) {
      double acc = x < nvec ? 0. : s[reflect101(x - r, w)] * k[0];
      for (int t = x < nvec ? 0 : 1; t < n; ++t) {
        const double v = s[reflect101(x + t - r, w)];
        acc = x < nvec ? fma(v, k[t], acc) : acc + v * k[t];
      }
      tmp[(size_t)y * w + x] = acc;
    }
  }
#pragma omp parallel for
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      double acc = tmp[(size_t)y * w + x] * k[r];
      for (int i = 1; i <= r; ++i)
        acc = acc + (tmp[(size_t)reflect101(y + i, h) * w + x] + tmp[(size_t)reflect101(y - i, h) * w + x]) * k[r + i];
      dst[(size_t)y * w + x] = acc;
    }
}

/* cv2.resize(src CV_64F 2-D, (ow, oh), INTER_LINEAR), both sides >= 2: source coordinate fma(d + 0.5, ssize / dsize, -0.5)
 * in double, i = floor, t = the rest; each pass is the lerp fma(b - a, t, a) of the two clamped taps, rows first. */
static void lin_taps_f64(int dsize, int ssize, int* i0, int* i1, double* t) {
  const double scale = (double)ssize / dsize;
  for (int d = 0; d < dsize; ++d) {
    const double f = fma(d + 0.5, scale, -0.5), fl = floor(f);
    const int i = (int)fl;
    t[d] = f - fl;
    i0[d] = i < 0 ? 0 : (i > ssize - 1 ? ssize - 1 : i);
    i1[d] = i + 1 < 0 ? 0 : (i + 1 > ssize - 1 ? ssize - 1 : i + 1);
  }
}

void resize_linear_f64_ref(const double* src, int h, int w, double* dst, int oh, int ow) {
  int* xi = malloc(sizeof(int) * 2 * (ow + oh));
  double* xt = malloc(sizeof(double) * (ow + oh));
  int *x0 = xi, *x1 = xi + ow, *y0 = xi + 2 * ow, *y1 = xi + 2 * ow + oh;
  double *tx = xt, *ty = xt + ow;
  lin_taps_f64(ow, w, x0, x1, tx);
  lin_taps_f64(oh, h, y0, y1, ty);
#pragma omp parallel for
  for (int y = 0; y < oh; ++y) {
    const double *r0 = src + (size_t)y0[y] * w, *r1 = src + (size_t)y1[y] * w;
    for (int x = 0; x < ow; ++x) {
      const double a = fma(r0[x1[x]] - r0[x0[x]], tx[x], r0[x0[x]]);
      const double b = fma(r1[x1[x]] - r1[x0[x]], tx[x], r1[x0[x]]);
      dst[(size_t)y * ow + x] = fma(b - a, ty[y], a);
    }
  }
  free(xi);
  free(xt);
}
