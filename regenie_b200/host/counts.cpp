#include "counts.hpp"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <thread>

namespace rgh {

void HardCallCounts::init(const ClassTable& ct, bool ref_first_, size_t n_file, const std::vector<int32_t>& sample_idx) {
  T = ct.T; binary = ct.binary; ref_first = ref_first_;
  words = (n_file + 31) / 32;
  m_all.assign((size_t)T * 2 * words, 0);
  m_male.assign((size_t)T * 2 * words, 0);
  const size_t N = sample_idx.size();
  for (int t = 0; t < T; ++t)
    for (size_t k = 0; k < N; ++k) {
      const int c = ct.cls[(size_t)t * N + k];
      if (!c) continue;
      const size_t f = (size_t)sample_idx[k];
      const uint64_t bit = 1ull << (2 * (f % 32));
      m_all[at(t, c - 1) + f / 32] |= bit;
      if (!ct.male.empty() && ct.male[k]) m_male[at(t, c - 1) + f / 32] |= bit;
    }
}

void HardCallCounts::count(const uint8_t* rows, size_t row_stride, int bs, const uint8_t* non_par, long* out, int threads) const {
  std::atomic<int> next{0};
  auto work = [&]() {
    std::vector<long> c((size_t)T * 2 * 6);                  // [column][class][all: het, two, none | male: het, two, none]
    for (;;) {
      const int v = next.fetch_add(1);
      if (v >= bs) return;
      const uint8_t* r = rows + (size_t)v * row_stride;
      const bool np = non_par && non_par[v];
      std::fill(c.begin(), c.end(), 0);
      for (size_t w = 0; w < words; ++w) {
        uint64_t x = 0;
        const size_t off = w * 8, nb = off + 8 <= row_stride ? 8 : row_stride - off;
        memcpy(&x, r + off, nb);                             // little endian: field s of the word = sample 32 w + s
        const uint64_t lo = x & 0x5555555555555555ull, hi = (x >> 1) & 0x5555555555555555ull;
        const uint64_t het = hi & ~lo, c11 = hi & lo, c00 = ~hi & ~lo & 0x5555555555555555ull;   // 01 = missing
        for (int tc = 0; tc < 2 * T; ++tc) {
          const uint64_t ma = m_all[(size_t)tc * words + w];
          if (!ma) continue;
          long* cc = &c[(size_t)tc * 6];
          cc[0] += __builtin_popcountll(het & ma); cc[1] += __builtin_popcountll(c00 & ma); cc[2] += __builtin_popcountll(c11 & ma);
          if (np) {
            const uint64_t mm = m_male[(size_t)tc * words + w];
            cc[3] += __builtin_popcountll(het & mm); cc[4] += __builtin_popcountll(c00 & mm); cc[5] += __builtin_popcountll(c11 & mm);
          }
        }
      }
      long* o = out + (size_t)v * T * 6;
      for (int t = 0; t < T; ++t)
        for (int k = 0; k < 2; ++k) {                         // k = 0: the "cases" columns, 1: the "controls" columns
          long* u = o + t * 6 + 3 * k;
          if (k == 1 && !binary) { u[0] = u[1] = u[2] = 0; continue; }
          const long* cc = &c[((size_t)t * 2 + (binary ? 1 - k : 0)) * 6];   // class 2 (cases) first for a binary column
          // PLINK 1 code 00 = two copies of the first .bim allele: the counted allele unless --ref-first
          const long het = cc[0], alt = ref_first ? cc[2] : cc[1], ref = ref_first ? cc[1] : cc[2];
          const long het_m = cc[3];
          u[0] = ref; u[1] = het - het_m; u[2] = alt + het_m;  // non-PAR males: g >= 1 -> alt (het_m = 0 elsewhere)
        }
    }
  };
  const int nt = std::max(1, std::min(threads, bs));
  std::vector<std::thread> pool;
  for (int t = 1; t < nt; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

void dosage_counts(const ClassTable& ct, bool ref_first, size_t n_file, const std::vector<int32_t>& sample_idx,
                   const uint8_t* probs, const uint8_t* pm, size_t n, const uint8_t* non_par, long* out, int threads) {
  const int T = ct.T;
  const bool binary = ct.binary;
  const uint8_t* cls = ct.cls.data();
  const uint8_t* male = ct.male.empty() ? nullptr : ct.male.data();
  std::atomic<size_t> next{0};
  const size_t nk = sample_idx.size();
  // samples per (column, class): the reference class follows by difference, so only het / alt / missing calls touch the columns
  std::vector<long> size((size_t)T * 3, 0);
  for (int t = 0; t < T; ++t)
    for (size_t k = 0; k < nk; ++k) ++size[(size_t)t * 3 + cls[(size_t)t * nk + k]];
  auto work = [&]() {
    std::vector<long> c((size_t)T * 3 * 3);                  // [column][class][het, alt, missing]
    for (;;) {
      const size_t j = next.fetch_add(1);
      if (j >= n) return;
      const uint8_t* pr = probs + j * n_file * 2;
      const uint8_t* m = pm + j * n_file;
      std::fill(c.begin(), c.end(), 0);
      for (size_t k = 0; k < nk; ++k) {
        const size_t f = (size_t)sample_idx[k];
        int g;
        if (m[f] & 0x80) g = 2;
        else {
          const uint32_t p0 = pr[2 * f], p1 = pr[2 * f + 1];
          const uint32_t hom = ref_first ? (p0 + p1 > 255 ? 0 : 255 - p0 - p1) : p0;
          const uint32_t d = p1 + 2 * hom;                   // dosage in units of 1 / 255
          if (male && non_par && non_par[j] && male[k]) {
            // dosage >= 1 is the one threshold an 8-bit pair can hit exactly (p1 + 2 hom = 255): decided in the reference's own
            // floating-point expression (parseSnpfromBGEN, src/Geno.cpp:2273-2281); the others (0.5, 1.5) cannot be hit
            const double a = p0 / 255.0, b = p1 / 255.0;
            const double val = ref_first ? b + 2 * std::max(1 - a - b, 0.0) : b + 2 * a;
            if (val >= 1) g = 1; else continue;
          }
          else if (2 * d >= 765) g = 1; else if (2 * d >= 255) g = 0; else continue;
        }
        for (int t = 0; t < T; ++t) ++c[((size_t)t * 3 + cls[(size_t)t * nk + k]) * 3 + g];
      }
      long* o = out + j * (size_t)T * 6;
      for (int t = 0; t < T; ++t) {
        const int first = binary ? 2 : 1;                    // class printed in the "cases" columns
        const long* a = &c[((size_t)t * 3 + first) * 3];
        o[t * 6 + 1] = a[0]; o[t * 6 + 2] = a[1]; o[t * 6 + 0] = size[(size_t)t * 3 + first] - a[0] - a[1] - a[2];
        const long* b = &c[((size_t)t * 3 + 1) * 3];
        o[t * 6 + 4] = binary ? b[0] : 0; o[t * 6 + 5] = binary ? b[1] : 0;
        o[t * 6 + 3] = binary ? size[(size_t)t * 3 + 1] - b[0] - b[1] - b[2] : 0;
      }
    }
  };
  const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)threads, n));
  std::vector<std::thread> pool;
  for (int t = 1; t < nt; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

}  // namespace rgh
