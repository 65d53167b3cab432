// Level-0 sufficient statistics on the tensor cores, exactly.
//
// The skinny products  G0 [X | Y]  and  Miss [X | Y]  per fold (A_f = G_f X_f and G_f Y_f of l0_stats.cu; the
// reference's `Gmat * new_cov`, src/Data.cpp:199, and `Gmat * phenotypes`, src/Data.cpp:746) are one more
// column tile of the same INT8 Gram kernel: the right operand is a fixed digit matrix D built ONCE per run from the
// covariate basis and the phenotypes,
//   xy[t, c] = (s_c / 15) * sum_l d_l[t, c] 30^-l,   d_l in {-15..15} (int8), 9 limbs = 44 bits,
// so each tensor-core product is an integer <= 240 (the planes carry 8), each fold sum an exact integer in the int32
// accumulators, and the FP64 Horner below reassembles  sum_t g(i,t) xy[t,c]  to ~5e-14 s_c per sample.
// A column of ones gives sum g0 and the missing count; together with the Gram diagonal (sum g0^2) that is n1, n2, nm.
// This replaces l0_stats_kernel + l0_fold_reduce_kernel (2.6e9 FP64 FMAs per block) by 22 % more Gram tiles.
#include "kernels.cuh"

namespace rg {

// digit rows of xy.  D: [drows][npad] bytes; row (c / 14) * 128 + (c % 14) * 9 + l; ones at row 126.
// grid: cpp (+1 for the ones row), block 256.
__global__ void __launch_bounds__(256)
l0_xy_digits_kernel(const double* __restrict__ xy, int cpp, int ncol, int64_t npad, const uint8_t* __restrict__ is_real,
                    double* __restrict__ scale, uint8_t* __restrict__ D) {
  __shared__ double red[256];
  const int c = blockIdx.x;
  if (c == ncol) {      // ones over the real (non-padding) samples
    uint8_t* row = D + (int64_t)kStatOnesRow * npad;
    for (int64_t t = threadIdx.x; t < npad; t += 256) row[t] = is_real[t] ? 0x01 : 0x00;
    return;
  }
  double mx = 0.0;
  for (int64_t t = threadIdx.x; t < npad; t += 256) mx = fmax(mx, fabs(xy[t * cpp + c]));
  mx = cta_tree<256, CtaOp::kMax>(mx, red);
  const double s = mx > 0.0 ? mx : 1.0;
  if (threadIdx.x == 0) scale[c] = s;
  uint8_t* base = D + ((int64_t)(c / kStatQ) * 128 + (c % kStatQ) * kLimbs) * npad;
  for (int64_t t = threadIdx.x; t < npad; t += 256) {
    double v = xy[t * cpp + c] / s * 15.0;
#pragma unroll
    for (int l = 0; l < kLimbs; ++l) {
      const double d = rint(v);
      const int di = (int)d;
      base[(int64_t)l * npad + t] = (uint8_t)(int8_t)di;
      v = (v - d) * 30.0;
    }
  }
}

// T [K][2 rows_p][ldt] exact integer sums -> cnt_fold [K][rows_p][4], sum_fold [K][rows_p][2][cpp].
// grid: (ceil(rows_p/128), K), block 128: thread = SNP row.
__global__ void __launch_bounds__(128)
l0_stats_finish_kernel(const float* __restrict__ T, int ldt, int64_t t_fold_stride, const float* __restrict__ zz,
                       int ldz, int64_t zz_fold_stride, int rows_p, int cpp, int ncol,
                       const double* __restrict__ scale, int32_t* __restrict__ cnt_fold,
                       double* __restrict__ sum_fold) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  const int f = blockIdx.y;
  if (i >= rows_p) return;
  const float* tg = T + (int64_t)f * t_fold_stride + (int64_t)i * ldt;
  const float* tm = T + (int64_t)f * t_fold_stride + (int64_t)(rows_p + i) * ldt;
  const int64_t per = (int64_t)rows_p * 2 * cpp;
  double* og = sum_fold + (int64_t)f * per + ((int64_t)i * 2) * cpp;
  double* om = og + cpp;
  for (int c = 0; c < cpp; ++c) {
    double a = 0.0, b = 0.0;
    if (c < ncol) {
      const int r0 = (c / kStatQ) * 128 + (c % kStatQ) * kLimbs;
#pragma unroll
      for (int l = kLimbs - 1; l >= 0; --l) {
        a = a * (1.0 / 30.0) + (double)tg[r0 + l];
        b = b * (1.0 / 30.0) + (double)tm[r0 + l];
      }
      const double s = scale[c] * (1.0 / 15.0);
      a *= s; b *= s;
    }
    og[c] = a;
    om[c] = b;
  }
  const int s1 = (int)tg[kStatOnesRow], nm = (int)tm[kStatOnesRow];
  const int s2 = (int)zz[(int64_t)f * zz_fold_stride + (int64_t)i * ldz + i];
  const int n2 = (s2 - s1) / 2, n1 = 2 * s1 - s2;
  reinterpret_cast<int4*>(cnt_fold)[(int64_t)f * rows_p + i] = make_int4(n1, n2, nm, 0);
}

void launch_l0_xy_digits(const double* xy, int cpp, int ncol, int64_t npad, const uint8_t* is_real, double* scale,
                         uint8_t* D, cudaStream_t s) {
  l0_xy_digits_kernel<<<ncol + 1, 256, 0, s>>>(xy, cpp, ncol, npad, is_real, scale, D);
}

void launch_l0_stats_finish(const float* T, int ldt, int64_t t_fold_stride, const float* zz, int ldz,
                            int64_t zz_fold_stride, int rows_p, int cpp, int ncol, int K, const double* scale,
                            int32_t* cnt_fold, double* sum_fold, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(rows_p, 128), K);
  l0_stats_finish_kernel<<<grid, 128, 0, s>>>(T, ldt, t_fold_stride, zz, ldz, zz_fold_stride, rows_p, cpp, ncol, scale,
                                              cnt_fold, sum_fold);
}

}  // namespace rg
