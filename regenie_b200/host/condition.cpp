#include "condition.hpp"

#include "textio.hpp"

namespace rgh {

void Conditioning::read_list() {
  LineReader fh(list_file);
  std::string line;
  while (fh.getline(line)) {
    const auto t = split_ws(line);
    if (t.empty()) throw Fail("incorrectly formatted file (" + list_file + ")");
    ids.insert(t[0]);                                        // duplicates count once
  }
  if (ids.size() > max_vars)
    throw Fail("number of variants used for conditional analysis is greater than maximum of " + std::to_string(max_vars) +
               " (otherwise use --max-condition-vars)");
  if (ids.empty()) throw Fail("no variants for conditional analysis given in file " + list_file);
}

// the variants of `ids` only; samples are matched by FID_IID afterwards, so the reader keeps all of them
void Conditioning::open_source(const std::string& f, const std::string& path, const std::string& sample,
                               const std::string& bgi, const std::set<int>& chrs) {
  src_fmt = f;
  if (f == "bgen") {
    bgen.reset(new BgenFile());
    bgen->open(path, sample, ref_first, {}, ids, {}, {}, chrs, bgi);
  } else {
    bed.reset(new BedFile());
    if (f == "pgen") bed->open_pgen(path, {}, ids, {}, {}, chrs);
    else bed->open(path, ref_first, {}, ids, {}, {}, chrs);
  }
}

void Conditioning::find(bool same_file, bool set_range, int range_chr, double range_min, double range_max) {
  const std::vector<Snp>& snps = bgen ? bgen->snps : bed->snps;
  std::map<std::string, size_t> at;                          // the last variant of an ID, like the reference's ID maps
  for (size_t j = 0; j < snps.size(); ++j) {
    const Snp& s = snps[j];
    if (set_range && (s.chrom != range_chr || (double)s.pos < range_min || (double)s.pos > range_max)) continue;
    at[s.id] = j;
  }
  rows.clear();
  for (const auto& id : ids) {
    auto it = at.find(id);
    if (it != at.end()) rows.push_back(it->second);
  }
  if (rows.empty())
    throw Fail(same_file ? "none of the variants were found in the genotype file" : "none of the conditional variants were found in the genotype file");
  if (rows.size() != ids.size())
    throw Fail(std::to_string(ids.size() - rows.size()) + " of the variants could not be found in the genotype file");
}

void Conditioning::locate_in_main(const std::string& main_fmt, const std::string& path, const std::string& sample,
                                  const std::string& bgi, const std::set<int>& chrs, bool set_range, int range_chr,
                                  double range_min, double range_max) {
  open_source(main_fmt, path, sample, bgi, chrs);
  find(true, set_range, range_chr, range_min, range_max);
}

void Conditioning::append(const SampleSet& g, Pheno& ph, Log& log) {
  const int64_t N = ph.N;
  if (external()) {                                          // extract_from_genofile (src/Geno.cpp:4217-4280)
    log << "    +conditioning on variants in [" << list_file << "]\n";
    log << (fmt == "bgen" ? "      -extracting variants from file [" : fmt == "pgen" ? "      -extracting variants using PGEN file prefix ["
                                                                                   : "      -extracting variants using BED file prefix [")
        << file << "]\n";
    open_source(fmt, file, sample_file, "", {});
  }
  // the samples of the source file that are analysed (setup_bed / setup_pgen / setup_bgen): the others are skipped, and
  // an analysed sample the file lacks is imputed like a missing call; the analysis sample set itself is left as it is
  const std::vector<std::string>& keys_file = bgen ? bgen->keys_file : bed->keys_file;
  std::vector<int64_t> to_kept(keys_file.size(), -1);
  bool any = false;
  for (size_t i = 0; i < keys_file.size(); ++i) {
    auto k = g.key_to_ind.find(keys_file[i]);
    if (k == g.key_to_ind.end() || !ph.in_cov[k->second]) continue;
    to_kept[i] = k->second;
    any = true;
  }
  if (external()) {
    if (!any) throw Fail("none of the analyzed samples are present in the file");
    find(false, false, 0, 0, 0);
    log << "      -n_used = " << ids.size() << "\n";
  } else {
    log << "    +conditioning on variants in [" << list_file << "] n_used = " << ids.size() << "\n";
  }
  const int K = (int)ids.size();
  if (ph.C + K > kMaxCovColumns)
    throw Fail("too many covariates for conditional analysis: " + std::to_string(ph.C) + " covariate columns (with the intercept) and " +
               std::to_string(K) + " conditioning variants make " + std::to_string(ph.C + K) + ", more than the maximum of " +
               std::to_string(kMaxCovColumns) + " columns");
  // read_snp / read_snps_* (src/Geno.cpp:3978-3996, :4367-4660): the genotype as the main reader codes it (allele count,
  // or the 8-bit dosage of a BGEN file), -3 = no call; the mean over the analysed samples with a call fills the gaps.
  // Its orientation (--ref-first) does not matter: the intercept is in the span.  The mean is formed from the integer
  // sum of the calls (allele counts, or dosages in units of 1/255), so it does not depend on the summation order.
  const size_t n_file = keys_file.size();
  std::vector<double> col(N);
  std::vector<uint8_t> row(bed ? bed->row_stride : 0), probs(bgen ? 2 * n_file : 0), pmiss(bgen ? n_file : 0);
  ph.X.resize((size_t)N * (ph.C + K));
  for (int c = 0; c < K; ++c) {
    std::fill(col.begin(), col.end(), -3.0);
    if (bgen) bgen->read_block(rows[c], 1, probs.data(), pmiss.data(), 1);
    else bed->read_rows(rows[c], 1, row.data());
    int64_t total = 0, ns = 0;
    for (size_t i = 0; i < n_file; ++i) {
      if (to_kept[i] < 0) continue;
      int v;
      if (bgen) {
        if (pmiss[i] & 0x80) continue;
        const int p0 = probs[2 * i], p1 = probs[2 * i + 1], p2 = p0 + p1 <= 255 ? 255 - p0 - p1 : 0;
        v = p1 + 2 * (ref_first ? p2 : p0);
      } else {
        // PLINK 1 codes 00 / 10 / 11 = two / one / no copies of the first .bim allele (ALT of a .pgen), 01 = missing
        const int code = (row[i >> 2] >> (2 * (i & 3))) & 3;
        if (code == 1) continue;
        const int cnt = code == 0 ? 2 : code == 2 ? 1 : 0;
        v = (ref_first && src_fmt == "bed") ? 2 - cnt : cnt;
      }
      col[to_kept[i]] = bgen ? v / 255.0 : v;
      total += v;
      ++ns;
    }
    if (ns > 0) {                                            // mean_impute_g (src/Geno.cpp:3190-3193)
      const double mu = (double)total / ((bgen ? 255.0 : 1.0) * (double)ns);
      for (int64_t s = 0; s < N; ++s) col[s] = !ph.in_cov[s] ? 0.0 : col[s] == -3.0 ? mu : col[s];
    }                                                        // no call at all: the column stays constant (-3)
    std::copy(col.begin(), col.end(), ph.X.begin() + (size_t)(ph.C + c) * N);
  }
  ph.C += K;
  bed.reset();                                               // the source reader (a .pgen is held in memory) is done
  bgen.reset();
}

}  // namespace rgh
