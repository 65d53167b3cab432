// Genotype counts of the Step-2 rows: N_RR / N_RA / N_AA of --no-split (print_sum_stats_all, src/Step2_Models.cpp:2441-2493)
// and Ref / Het / Alt per trait of --htp (update_genocounts, src/Geno.cpp:2986-3018), counted on the host from a block's
// bytes as the fetch thread read them: 2-bit rows (.bed, host-decoded .pgen) or 8-bit probability pairs (.bgen).
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace rgh {

// Which kept samples each of T columns counts, and how.  cls [T][kept samples]: 0 = not counted, 1 = counted (a control
// of a binary column), 2 = a case.  Both counters write out [bs][T][6]: ref / het / alt of class 2 then of class 1 for a
// binary column, of class 1 then three zeros otherwise.  Missing calls are not counted.  With a male vector [kept samples]
// and non-PAR flags [bs], a male call on the non-PAR part of chromosome X counts as alt when g >= 1 and as ref otherwise.
struct ClassTable {
  int T = 0;
  bool binary = false;
  std::vector<uint8_t> cls;
  std::vector<uint8_t> male;                                 // empty: no male rule
};

// Hard calls: per (column, class) a sample mask in FILE order with one bit per 2-bit field, three popcounts per 32 samples.
struct HardCallCounts {
  int T = 0;
  bool binary = false, ref_first = false;
  size_t words = 0;
  std::vector<uint64_t> m_all, m_male;                       // [T][2 classes][words]
  size_t at(int t, int c) const { return ((size_t)t * 2 + c) * words; }
  void init(const ClassTable& ct, bool ref_first, size_t n_file, const std::vector<int32_t>& sample_idx);
  // rows [bs][row_stride]; non_par [bs] or null
  void count(const uint8_t* rows, size_t row_stride, int bs, const uint8_t* non_par, long* out, int threads) const;
};

// Dosages: probs [n][n_file][2] and ploidy / missing bytes pm [n][n_file] as BgenFile::read_block inflates them;
// dosage >= 1.5 alt, >= 0.5 het.  non_par [n] or null.
void dosage_counts(const ClassTable& ct, bool ref_first, size_t n_file, const std::vector<int32_t>& sample_idx,
                   const uint8_t* probs, const uint8_t* pm, size_t n, const uint8_t* non_par, long* out, int threads);

}  // namespace rgh
