// Step-2 statistics for 8-bit BGEN dosages and the binary-trait (logistic) score test.
// Replaces, per variant: parseSnpfromBGEN (reference src/Geno.cpp:2186-2345: dosage = p1/255 + 2 p0/255,
// INFO numerator 4 p0 + p1 - g^2, AF / N / MAC), flip_geno (:3150), mean imputation, check_sparse_G (:3165)
// and compute_score_bt (src/Step2_Models.cpp:470-556).
//
// As for hard calls (s2_kernels.cu) every statistic is a linear/quadratic form of code-wise sums of a
// per-sample feature row F; with dosages the "codes" are the integers d = p1 + 2 p0 (0..510) and
// e = 4 p0 + p1, so the kernel accumulates  S1 = sum d F,  S2 = sum d^2 F,  Sm = sum miss F,  Se = sum e F
// and the finish is closed form - including the minor-allele flip and the imputed mean, which are
// affine in d.  Feature row for binary traits (per trait p):
//   F = [ a | m_p | w_p^2 | w_p yres_p | w_p XW_pc (C) ]      w_p = Gamma_p^{1/2} m_p
#include "kernels.cuh"

namespace rg {

constexpr int kDzCols = 16;
constexpr int kDzSub = 128;

// BGEN probability rows [bs][n_file][2] (+ optional ploidy/missing bytes [bs][n_file]) -> padded sample
// layout, one genotype word dz per sample (kernels.cuh).
__device__ __forceinline__ uint32_t dosage_word(uint32_t p0, uint32_t p1, bool m, int ref_first) {
  if (m) return kDzMissing;
  // ref-last: g = p1 + 2 p0 (allele0 is ALT);  ref-first: g = p1 + 2 p2, p2 = 255 - p0 - p1 (>= 0)
  const uint32_t p2 = (p0 + p1 <= 255u) ? 255u - p0 - p1 : 0u;
  const uint32_t hom = ref_first ? p2 : p0;
  return dz_word(p1 + 2u * hom, 4u * hom + p1);
}

// grid: (Npad/1024, rows_p), block 256: four consecutive padded samples per thread.  Almost every quad maps to four
// CONSECUTIVE samples of the file row (folds only shift ranges, --remove breaks a quad here and there): those take one
// 8-byte probability load, one 4-byte ploidy load and one 16-byte store when the addresses are aligned.
__global__ void dosage_relayout_kernel(const uint8_t* __restrict__ probs, const uint8_t* __restrict__ miss,
                                       int64_t n_file, int bs, const int32_t* __restrict__ file_idx_pad,
                                       int ref_first, uint32_t* __restrict__ dz, int64_t npad) {
  const int64_t t = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 4;
  const int row = blockIdx.y;
  if (t >= npad) return;
  uint4 out = make_uint4(0u, 0u, 0u, 0u);
  if (row < bs) {
    const int4 f = *reinterpret_cast<const int4*>(file_idx_pad + t);
    const int64_t e0 = (int64_t)row * n_file + f.x;
    if (f.x >= 0 && f.y == f.x + 1 && f.z == f.x + 2 && f.w == f.x + 3 &&
        (reinterpret_cast<uintptr_t>(probs + e0 * 2) & 7) == 0 && (!miss || (reinterpret_cast<uintptr_t>(miss + e0) & 3) == 0)) {
      const uint2 pr = *reinterpret_cast<const uint2*>(probs + e0 * 2);
      const uint32_t mm = miss ? *reinterpret_cast<const uint32_t*>(miss + e0) : 0u;
      out.x = dosage_word(pr.x & 0xFFu, (pr.x >> 8) & 0xFFu, (mm & 0x80u) != 0, ref_first);
      out.y = dosage_word((pr.x >> 16) & 0xFFu, pr.x >> 24, (mm & 0x8000u) != 0, ref_first);
      out.z = dosage_word(pr.y & 0xFFu, (pr.y >> 8) & 0xFFu, (mm & 0x800000u) != 0, ref_first);
      out.w = dosage_word((pr.y >> 16) & 0xFFu, pr.y >> 24, (mm & 0x80000000u) != 0, ref_first);
    } else {
      const int fi[4] = {f.x, f.y, f.z, f.w};
      uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (fi[k] < 0) continue;
        const uint8_t* pr = probs + ((int64_t)row * n_file + fi[k]) * 2;
        const bool m = miss ? (miss[(int64_t)row * n_file + fi[k]] & 0x80) != 0 : false;
        o[k] = dosage_word(pr[0], pr[1], m, ref_first);
      }
      out = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
  *reinterpret_cast<uint4*>(dz + (int64_t)row * npad + t) = out;
}

// S1 / S2 / Sm / Se partial sums of one chunk of samples for 64 variant rows x 16 feature columns, plus the non-zero /
// hom-alt counts check_sparse_G needs (analysed, non-missing samples with d != 0 resp. d == 510).
//   grid: (rows_p/64, nchunks, ceil(ncol/16)); block 64 x (live column groups, <= 4): thread = (variant row, 4 of the 16
//   columns).  part: [chunk][row][4][dp]
// Both operands of a 64-sample sub-tile go through shared memory: the feature rows (broadcast to every variant row, as before)
// and the dz words of the 64 rows, loaded with coalesced 256-byte row segments (the first version read them per thread with
// a stride of one whole row: 592 us per 400 variants at N = 100k, ~10x its FP64 bound; four threads per row also quadruple
// the warps that feed the FP64 pipe).  Summation order per (row, column): samples ascending inside the chunk; chunks are
// added in order by partial_sum_kernel - fixed, independent of the launch shape.
constexpr int kDzRows = 64;
constexpr int kDzSubS = 64;

__global__ void __launch_bounds__(256)
dosage_stats_kernel(const uint32_t* __restrict__ dz, int64_t npad, const double* __restrict__ F, int dp, int ncol,
                    const int4* __restrict__ chunks, int rows_p, double* __restrict__ part, int2* __restrict__ part_cnt) {
  __shared__ double2 tile[kDzSubS][kDzCols / 2];          // 8 KiB
  __shared__ uint32_t dzs[kDzRows][kDzSubS + 1];          // 16.25 KiB
  // variant row of the tile, column group (4 columns).  The column group is WARP-uniform (two warps per group), so the
  // groups beyond the last used column (ncol of the dp padded columns: 6 of 16 for one binary trait) cost nothing
  const int r = threadIdx.x & 63, cg = threadIdx.x >> 6;
  const int row0 = blockIdx.x * kDzRows;
  const int4 ch = chunks[blockIdx.y];
  const int col0 = blockIdx.z * kDzCols;
  const bool counter = blockIdx.z == 0 && cg == 0;        // this thread sees column 0 = the analysed-sample indicator
  double a1[4], a2[4], am[4], ae[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) a1[c] = a2[c] = am[c] = ae[c] = 0.0;
  int nz = 0, n510 = 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool live = col0 + 4 * cg < ncol;
  for (int sub = 0; sub < ch.y; sub += kDzSubS) {
    const int t0 = ch.x + sub;
    __syncthreads();
    for (int e = threadIdx.x; e < kDzSubS * (kDzCols / 2); e += blockDim.x) {
      const int s = e / (kDzCols / 2), c2 = e % (kDzCols / 2);
      tile[s][c2] = *reinterpret_cast<const double2*>(F + (int64_t)(t0 + s) * dp + col0 + 2 * c2);
    }
    for (int rr = warp; rr < kDzRows; rr += (int)(blockDim.x >> 5)) {   // one row segment (64 words) per warp pass, two words per lane
      const uint2 v2 = *reinterpret_cast<const uint2*>(dz + (int64_t)(row0 + rr) * npad + t0 + 2 * lane);
      dzs[rr][2 * lane] = v2.x;
      dzs[rr][2 * lane + 1] = v2.y;
    }
    __syncthreads();
    if (!live) continue;
#pragma unroll 4
    for (int s = 0; s < kDzSubS; ++s) {
      const uint32_t v = dzs[r][s];
      if (v == 0u) continue;
      const double2 f0 = tile[s][2 * cg], f1 = tile[s][2 * cg + 1];
      if (dz_missing(v)) {
        am[0] += f0.x; am[1] += f0.y; am[2] += f1.x; am[3] += f1.y;
      } else {
        const uint32_t di = dz_d(v);
        const double d = (double)di, e = (double)dz_e(v), d2 = d * d;
        a1[0] = fma(d, f0.x, a1[0]);  a1[1] = fma(d, f0.y, a1[1]);  a1[2] = fma(d, f1.x, a1[2]);  a1[3] = fma(d, f1.y, a1[3]);
        a2[0] = fma(d2, f0.x, a2[0]); a2[1] = fma(d2, f0.y, a2[1]); a2[2] = fma(d2, f1.x, a2[2]); a2[3] = fma(d2, f1.y, a2[3]);
        ae[0] = fma(e, f0.x, ae[0]);  ae[1] = fma(e, f0.y, ae[1]);  ae[2] = fma(e, f1.x, ae[2]);  ae[3] = fma(e, f1.y, ae[3]);
        if (counter && f0.x != 0.0) { nz += di != 0u; n510 += di == 510u; }
      }
    }
  }
  const int row = row0 + r;
  double* o = part + (((int64_t)blockIdx.y * rows_p + row) * 4) * dp + col0 + 4 * cg;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    o[c] = a1[c];
    o[dp + c] = a2[c];
    o[2 * dp + c] = am[c];
    o[3 * dp + c] = ae[c];
  }
  if (counter) part_cnt[(int64_t)blockIdx.y * rows_p + row] = make_int2(nz, n510);
}

// non-zero / hom-alt counts: fixed-order sum of the chunk counts.  grid: ceil(rows_p / 256)
__global__ void dosage_count_reduce_kernel(const int2* __restrict__ part_cnt, int nchunks, int rows_p, double* __restrict__ out,
                                           double* __restrict__ out510) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= rows_p) return;
  long long a = 0, b = 0;
  for (int c = 0; c < nchunks; ++c) {
    const int2 v = part_cnt[(int64_t)c * rows_p + row];
    a += v.x; b += v.y;
  }
  out[row] = (double)a;
  out510[row] = (double)b;
}

// one thread per variant: AF / INFO / N / MAC, flip, sparse switch and the BT score test.
__global__ void s2_bt_finalize_kernel(S2BtFinalizeArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.bs) return;
  const int C = a.C, P = a.P, dp = a.dp;
  const double* S1 = a.sums + ((int64_t)i * 4) * dp;
  const double* S2 = S1 + dp;
  const double* Sm = S1 + 2 * dp;
  const double* Se = S1 + 3 * dp;
  const double k = 1.0 / a.unit, k2 = k * k;
  const double nm = Sm[0];
  const bool xmale = a.non_par && a.non_par[i] && a.col_male >= 0;       // non-PAR chrX: see s2_count
  const S2Count all = s2_count(S1, S2, Sm, Se, 0, (double)a.n_analyzed, xmale ? a.col_male : -1,
                               a.col_tot + a.col_male, k, a.ns_all + i, a.mac_all + i, a.af_all + i, nullptr);
  const double ns1 = all.ns, total = S1[0] * k;       // dosage sum over analysed, non-missing samples
  int flags = 0;
  if (all.mac < a.min_mac) flags |= 1;
  double mu = total / ns1;
  const bool flip = a.with_flip && (mu > 1.0);        // flip_geno, src/Geno.cpp:3150-3163
  if (flip) { flags |= 8; mu = 2.0 - mu; }
  // non-zero entries among analysed samples after flip + imputation (check_sparse_G): a dosage is non-zero
  // iff d != 0, after a flip iff d != 510; imputed entries are non-zero iff the mean is.
  const double nnz = (flip ? ns1 - a.n510[i] : a.nz_count[i]) + ((mu != 0.0) ? nm : 0.0);
  const bool sparse = nnz <= (double)a.n_samples * 0.5;
  if (sparse) flags |= 4;
  a.scale_fac[i] = 1.0;
  a.flags[i] = flags;
  a.mu[i] = mu;
  for (int p = 0; p < P; ++p) {
    const int base = 1 + p * (3 + C);                 // [m_p | w^2 | w yres | w XW_c ...]
    const int64_t ip = (int64_t)i * P + p;
    s2_count(S1, S2, Sm, Se, base, a.col_tot[base], xmale ? a.col_male + 1 + p : -1,
             a.col_tot + a.col_male + 1 + p, k, a.ns + ip, a.mac + ip, a.af + ip, a.info + ip);
    // g_imp = (flip ? 2 - g : g) on non-missing, mu on missing.  For a feature f:
    //   sum g_imp f   = flip ? 2 (T - M) - s1 : s1,  + mu M      (T = sum f over analysed, M = sum over missing)
    //   sum g_imp^2 f = flip ? 4 (T - M) - 4 s1 + s2 : s2,  + mu^2 M
    auto lin = [&](int col) {
      const double s1 = S1[col] * k, M = Sm[col], T = a.col_tot[col];
      return (flip ? 2.0 * (T - M) - s1 : s1) + mu * M;
    };
    const int cw2 = base + 1, cwy = base + 2, cwx = base + 3;
    const double s1w2 = S1[cw2] * k, s2w2 = S2[cw2] * k2, Mw2 = Sm[cw2], Tw2 = a.col_tot[cw2];
    const double gw2 = (flip ? 4.0 * (Tw2 - Mw2) - 4.0 * s1w2 + s2w2 : s2w2) + mu * mu * Mw2;   // |GW|^2
    double xt2 = 0.0, xty = 0.0;
    for (int c = 0; c < C; ++c) {
      const double v = lin(cwx + c);                  // (XW^T GW)_c
      a.xtwg[((int64_t)i * P + p) * C + c] = v;
      xt2 += v * v;
      xty += v * a.xwy[(int64_t)p * C + c];           // (XW^T yres)_c
    }
    const double den = gw2 - xt2;                     // = |GW - XW XW^T GW|^2  (XW orthonormal)
    a.den[(int64_t)i * P + p] = den;
    double num = lin(cwy);                            // GW . yres
    if (!sparse) num -= xty;                          // dense path projects the covariates out of G first (:500,:521)
    const double sq = sqrt(den);
    double st = num / sq;
    if (!(sq >= a.numtol)) { st = 0.0; a.flags[i] |= 16; }
    const double se = 1.0 / sq;
    double beta = st * se;
    if (flip) beta = -beta;
    a.stat[(int64_t)i * P + p] = st;
    a.beta[(int64_t)i * P + p] = beta;
    a.se[(int64_t)i * P + p] = se;
    a.chisq[(int64_t)i * P + p] = st * st;
  }
}

__global__ void dosage_scale_kernel(const double* __restrict__ s4, int rows_p, int dp, double* __restrict__ s3,
                                    double* __restrict__ se) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= (int64_t)rows_p * dp) return;
  const int64_t r = e / dp, c = e % dp;
  const double k = 1.0 / 255.0;
  const double* in = s4 + (r * 4) * dp + c;
  double* o = s3 + (r * 3) * dp + c;
  o[0] = in[0] * k;
  o[dp] = in[dp] * k * k;
  o[2 * dp] = in[2 * dp];
  se[r * dp + c] = in[3 * dp] * k;
}

void launch_dosage_scale(const double* sums4, int rows_p, int dp, double* sums3, double* se, cudaStream_t s) {
  dosage_scale_kernel<<<(unsigned)ceil_div((int64_t)rows_p * dp, 256), 256, 0, s>>>(sums4, rows_p, dp, sums3, se);
}

void launch_dosage_relayout(const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs, int rows_p,
                            const int32_t* file_idx_pad, int ref_first, uint32_t* dz, int64_t npad, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(npad, 1024), rows_p);
  dosage_relayout_kernel<<<grid, 256, 0, s>>>(probs, miss, n_file, bs, file_idx_pad, ref_first, dz, npad);
}

void launch_dosage_stats(const uint32_t* dz, int64_t npad, const double* F, int dp, const int4* chunks, int nchunks,
                         int rows_p, double* part, int2* part_cnt, double* sums, double* nnz, double* n510, cudaStream_t s,
                         int ncol) {
  RG_CHECK(rows_p % kDzRows == 0 && dp % kDzCols == 0, "dosage statistics: rows_p % 64 == 0 and dp % 16 == 0");
  if (ncol <= 0 || ncol > dp) ncol = dp;
  dim3 grid(rows_p / kDzRows, nchunks, (unsigned)ceil_div(ncol, kDzCols));
  // threads only for the column groups (of 4) that hold used columns: one binary trait with 3 covariates has 7 of 16
  const int groups = grid.z > 1 ? 4 : (int)ceil_div(ncol, 4);
  if ((int)grid.z * kDzCols < dp || groups < 4) RG_CUDA(cudaMemsetAsync(part, 0, (size_t)nchunks * rows_p * 4 * dp * sizeof(double), s));
  dosage_stats_kernel<<<grid, 64 * groups, 0, s>>>(dz, npad, F, dp, ncol, chunks, rows_p, part, part_cnt);
  launch_partial_sum(part, nchunks, (int64_t)rows_p * 4 * dp, sums, s);
  dosage_count_reduce_kernel<<<(unsigned)ceil_div(rows_p, 256), 256, 0, s>>>(part_cnt, nchunks, rows_p, nnz, n510);
}

void launch_s2_bt_finalize(const S2BtFinalizeArgs& a, cudaStream_t s) {
  s2_bt_finalize_kernel<<<(unsigned)ceil_div(a.bs, 128), 128, 0, s>>>(a);
}

}  // namespace rg
