#include "data.hpp"

#include <fcntl.h>
#include <unistd.h>
#include <thread>
#include "textio.hpp"

#include <algorithm>
#include <cstring>

namespace rgh {

std::set<std::string> read_id_list(const std::string& path, int ncols) {
  std::set<std::string> out;
  if (path.empty()) return out;
  LineReader fh(path);
  std::string line;
  while (fh.getline(line)) {
    auto t = split_ws(line);
    if ((int)t.size() < ncols) continue;
    out.insert(ncols == 2 ? t[0] + "_" + t[1] : t[0]);
  }
  return out;
}

void BedFile::open(const std::string& pfx, bool ref_first, const std::set<std::string>& exclude,
                   const std::set<std::string>& extract, const std::set<std::string>& remove,
                   const std::set<std::string>& keep, const std::set<int>& chrs) {
  prefix = pfx;
  // ---- .bim
  {
    LineReader fh(prefix + ".bim");
    std::string line;
    uint64_t lineno = 0;
    int last_chr = 0;
    std::vector<int> chr_seen;
    while (fh.getline(line)) {
      auto t = split_ws(line);
      if (t.size() < 6) throw Fail("incorrectly formatted bim file at line " + std::to_string(lineno + 1));
      Snp s;
      s.chrom = chr_str_to_int(t[0]);
      if (s.chrom == -1) throw Fail("unknown chromosome code in bim file at line " + std::to_string(lineno + 1));
      if (chr_seen.empty() || chr_seen.back() != s.chrom) {
        if (s.chrom <= last_chr) throw Fail("chromosomes in bim file are not in ascending order.");
        chr_seen.push_back(s.chrom);
        last_chr = s.chrom;
      }
      s.id = t[1];
      s.pos = std::stoull(t[3], nullptr, 0);
      if (ref_first) { s.allele0 = t[4]; s.allele1 = t[5]; }
      else           { s.allele0 = t[5]; s.allele1 = t[4]; }
      s.offset = lineno++;
      if (!chrs.empty() && !chrs.count(s.chrom)) continue;          // --chr / --chrList (in_chrList, src/Geno.cpp)
      if (exclude.count(s.id)) continue;
      if (!extract.empty() && !extract.count(s.id)) continue;
      snps.push_back(s);
    }
  }
  // ---- .fam
  {
    LineReader fh(prefix + ".fam");
    std::string line;
    std::set<std::string> seen;
    while (fh.getline(line)) {
      auto t = split_ws(line);
      if (t.empty()) continue;
      if (t.size() < 6) throw Fail("incorrectly formatted fam file.");
      const std::string k = t[0] + "_" + t[1];
      if (!seen.insert(k).second) throw Fail("duplicate individual in fam file : FID_IID=" + k);
      keys_file.push_back(k);
      ids_file.emplace_back(t[0], t[1]);
      sex_file.push_back((t[4] == "1") ? 1 : (t[4] == "2" ? 2 : 0));
    }
  }
  for (size_t i = 0; i < keys_file.size(); ++i) {
    const std::string& k = keys_file[i];
    if (remove.count(k)) continue;
    if (!keep.empty() && !keep.count(k)) continue;
    if (sex_specific && sex_file[i] != sex_specific) continue;   // --sex-specific (src/Geno.cpp:1287-1293)
    key_to_ind[k] = (uint32_t)keys.size();
    keys.push_back(k);
    sample_idx.push_back((int32_t)i);
  }
  if (keys.empty()) throw Fail("no samples left after --keep/--remove/--sex-specific.");
  row_stride = (keys_file.size() + 3) / 4;
  // ---- .bed
  bed.open(prefix + ".bed", std::ios::binary);
  if (!bed) throw Fail("cannot open file : " + prefix + ".bed");
  unsigned char magic[3];
  bed.read(reinterpret_cast<char*>(magic), 3);
  if (!(magic[0] == 0x6c && magic[1] == 0x1b && magic[2] == 0x01))
    throw Fail("invalid bed file (expected SNP-major mode, magic 6c 1b 01).");
  bed_fd = ::open((prefix + ".bed").c_str(), O_RDONLY);
}

BedFile::~BedFile() {
  if (bed_fd >= 0) ::close(bed_fd);
}

// n bytes at file offset off, on up to 8 threads when the run is long (a 1000-SNP block at N = 100k is 25 MB: one thread
// copies it out of the page cache in ~5 ms, which would bound level 0 from a file)
static void pread_all(int fd, uint8_t* dst, size_t n, uint64_t off) {
  auto part = [fd](uint8_t* d, size_t len, uint64_t o) {
    while (len) {
      const ssize_t r = ::pread(fd, d, len, (off_t)o);
      if (r <= 0) throw Fail("cannot read from bed file.");
      d += r; o += (uint64_t)r; len -= (size_t)r;
    }
  };
  const size_t T = n >= (8u << 20) ? std::min<size_t>(8, std::max(1u, std::thread::hardware_concurrency())) : 1;
  if (T == 1) { part(dst, n, off); return; }
  const size_t step = (n / T + 4095) / 4096 * 4096;
  std::vector<std::thread> pool;
  std::vector<std::string> errs(T);
  for (size_t t = 0; t < T; ++t) {
    const size_t lo = std::min(n, t * step), hi = std::min(n, lo + step);
    if (lo == hi) continue;
    pool.emplace_back([&, t, lo, hi] { try { part(dst + lo, hi - lo, off + lo); } catch (const std::exception& e) { errs[t] = e.what(); } });
  }
  for (auto& th : pool) th.join();
  for (auto& e : errs) if (!e.empty()) throw Fail(e);
}

void pgen_read_rows(PgenFile& pg, size_t first, size_t n, uint8_t* out);

void BedFile::read_rows(size_t first, size_t n, uint8_t* out) {
  if (pg) { pgen_read_rows(*pg, first, n, out); return; }
  // runs of consecutive file rows (the common case: no --extract holes) are read with one call
  size_t j = 0;
  while (j < n) {
    size_t e = j + 1;
    while (e < n && snps[first + e].offset == snps[first + e - 1].offset + 1) ++e;
    if (bed_fd >= 0) {
      pread_all(bed_fd, out + j * row_stride, (e - j) * row_stride, 3 + snps[first + j].offset * row_stride);
    } else {
      bed.seekg(3 + snps[first + j].offset * row_stride, std::ios::beg);
      bed.read(reinterpret_cast<char*>(out + j * row_stride), (std::streamsize)((e - j) * row_stride));
      if (!bed) throw Fail("cannot read from bed file.");
    }
    j = e;
  }
}

// [n x k] table keyed by FID_IID; samples absent from the genotype file are ignored
static void read_table(const std::string& path, const SampleSet& g, const std::set<std::string>* skip_cols,
                       const std::set<std::string>* only_cols, std::vector<std::string>& names,
                       const std::set<std::string>* cat_cols, std::vector<std::map<std::string, int>>* cat_levels, std::vector<double>& vals, std::vector<uint8_t>& present) {
  LineReader fh(path);
  std::string line;
  fh.getline(line);
  auto hdr = split_ws(line);
  if (hdr.size() < 2 || hdr[0] != "FID" || hdr[1] != "IID") throw Fail("header of file must start with: FID IID.");
  std::vector<int> keep;
  for (size_t i = 2; i < hdr.size(); ++i)
    if ((!skip_cols || !skip_cols->count(hdr[i])) && (!only_cols || only_cols->empty() || only_cols->count(hdr[i]))) {
      keep.push_back((int)i);
      names.push_back(hdr[i]);
    }
  if (only_cols)                                           // --phenoCol / --covarCol name a column that must exist
    for (const auto& c : *only_cols)
      if (std::find(hdr.begin() + 2, hdr.end(), c) == hdr.end()) throw Fail("column '" + c + "' was not found in file : " + path);
  const size_t n = g.keys.size(), k = keep.size();
  if (cat_levels) cat_levels->assign(k, {});
  vals.assign(n * k, 0.0);
  present.assign(n, 0);
  while (fh.getline(line)) {
    auto t = split_ws(line);
    if (t.empty()) continue;
    if (t.size() != hdr.size()) throw Fail("incorrectly formatted file : " + path);
    auto it = g.key_to_ind.find(t[0] + "_" + t[1]);
    if (it == g.key_to_ind.end()) continue;
    const size_t s = it->second;
    if (present[s]) throw Fail("individual appears more than once in file: FID=" + t[0] + " IID=" + t[1]);
    present[s] = 1;
    for (size_t c = 0; c < k; ++c) {
      const std::string& tok = t[keep[c]];
      if (cat_cols && cat_cols->count(names[names.size() - k + c])) {        // categorical: level index, NA stays missing
        if (tok == "NA") { vals[c * n + s] = kMissing; continue; }
        auto& lv = (*cat_levels)[c];
        auto it = lv.find(tok);
        if (it == lv.end()) it = lv.emplace(tok, (int)lv.size()).first;
        vals[c * n + s] = (double)it->second;
      } else {
        vals[c * n + s] = convert_double(tok);
      }
    }
  }
}

void read_pheno_and_cov(const SampleSet& g, const std::string& pheno_file, const std::string& covar_file,
                        bool step2, bool strict, bool bt, Pheno& ph, Log& log) {
  const int64_t N = (int64_t)g.keys.size();
  ph.N = N;
  ph.bt = bt;
  ph.step1 = !step2;
  std::vector<uint8_t> in_ph;
  read_table(pheno_file, g, ph.pheno_excl.empty() ? nullptr : &ph.pheno_excl, &ph.pheno_cols, ph.names, nullptr, nullptr, ph.Y, in_ph);
  ph.P = (int)ph.names.size();
  if (ph.P < 1) throw Fail("need at least one phenotype.");
  log << " * phenotypes          : [" << pheno_file << "] n_pheno = " << ph.P << "\n";
  ph.strict = strict || ph.P == 1;                          // src/Pheno.cpp:198
  ph.mask.assign((size_t)N * ph.P, 1);
  if (bt) {                                                 // src/Pheno.cpp:296-315: controls 0, cases 1, else NA
    ph.Y_raw = ph.Y;
    for (size_t e = 0; e < ph.Y_raw.size(); ++e) {
      const double y = ph.Y_raw[e];
      if (y == 0.0 || y == 1.0) continue;
      if (y != kMissing) throw Fail("a phenotype value is not 0/1/NA for a binary trait.");
      ph.mask[e] = 0;
    }
  }
  for (int64_t s = 0; s < N; ++s) {
    bool all_miss = true, any_miss = false;
    for (int p = 0; p < ph.P; ++p) {
      const bool miss = ph.Y[(size_t)p * N + s] == kMissing;
      if (!miss) all_miss = false; else any_miss = true;
      if (miss && step2 && !bt) ph.mask[(size_t)p * N + s] = 0;   // rm_missing_qt (src/Pheno.cpp:331)
    }
    if (ph.strict && any_miss) {
      for (int p = 0; p < ph.P; ++p) ph.mask[(size_t)p * N + s] = 0;
      all_miss = true;
    }
    if (all_miss) in_ph[s] = 0;
    if (!in_ph[s]) for (int p = 0; p < ph.P; ++p) ph.mask[(size_t)p * N + s] = 0;
  }
  // every trait needs at least one observation (src/Pheno.cpp:343-351)
  {
    std::vector<int64_t> nobs(ph.P, 0);
    for (int p = 0; p < ph.P; ++p)
      for (int64_t s = 0; s < N; ++s) nobs[p] += ph.mask[(size_t)p * N + s];
    if (std::all_of(nobs.begin(), nobs.end(), [](int64_t n) { return n == 0; }))
      throw Fail("all individuals have missing/invalid values for all traits.");
    for (int p = 0; p < ph.P; ++p)
      if (nobs[p] == 0) throw Fail("all individuals have missing/invalid values for phenotype '" + ph.names[p] + "'.");
  }
  // binary traits with fewer than --minCaseCount cases are dropped (rm_phenoCols, src/Pheno.cpp:527-570)
  if (bt) {
    std::vector<int> keep;
    for (int p = 0; p < ph.P; ++p) {
      int64_t cases = 0;
      for (int64_t s = 0; s < N; ++s) cases += ph.Y_raw[(size_t)p * N + s] == 1.0;
      if (cases >= ph.min_case_count) keep.push_back(p);
    }
    if (keep.empty()) throw Fail("all phenotypes have less than " + std::to_string(ph.min_case_count) + " cases.");
    if ((int)keep.size() < ph.P) {
      log << "   -removing phenotypes with fewer than " << ph.min_case_count << " cases\n";
      for (int p = 0, k = 0; p < ph.P; ++p) {
        if (k < (int)keep.size() && keep[k] == p) { ++k; continue; }
        log << "    +WARNING: Phenotype '" << ph.names[p] << "' has too few cases so it will be ignored.\n";
      }
      std::vector<std::string> names;
      std::vector<double> Y, Yr;
      std::vector<uint8_t> mask;
      for (int p : keep) {
        names.push_back(ph.names[p]);
        Y.insert(Y.end(), ph.Y.begin() + (size_t)p * N, ph.Y.begin() + (size_t)(p + 1) * N);
        Yr.insert(Yr.end(), ph.Y_raw.begin() + (size_t)p * N, ph.Y_raw.begin() + (size_t)(p + 1) * N);
        mask.insert(mask.end(), ph.mask.begin() + (size_t)p * N, ph.mask.begin() + (size_t)(p + 1) * N);
      }
      ph.names.swap(names); ph.Y.swap(Y); ph.Y_raw.swap(Yr); ph.mask.swap(mask);
      ph.P = (int)keep.size();
      for (int64_t s = 0; s < N; ++s) {                      // samples left without any phenotype value
        bool any = false;
        for (int p = 0; p < ph.P; ++p) any |= ph.mask[(size_t)p * N + s] != 0;
        if (!any) in_ph[s] = 0;
      }
      log << "    + n_pheno = " << ph.P << "\n";
    }
  }
  // covariates: intercept first (src/Pheno.cpp:79)
  std::vector<uint8_t> in_cov(N, 1);
  std::vector<double> cov;
  std::vector<std::string> cnames;
  if (!covar_file.empty()) {
    std::set<std::string> skip(ph.names.begin(), ph.names.end());
    skip.insert(ph.covar_excl.begin(), ph.covar_excl.end());
    std::set<std::string> only = ph.covar_cols;
    if (!only.empty()) only.insert(ph.cat_cols.begin(), ph.cat_cols.end());   // --catCovarList columns are covariates too
    std::vector<std::map<std::string, int>> levels;
    read_table(covar_file, g, &skip, &only, cnames, &ph.cat_cols, &levels, cov, in_cov);
    for (const auto& c : ph.cat_cols)
      if (std::find(cnames.begin(), cnames.end(), c) == cnames.end()) throw Fail("column '" + c + "' was not found in file : " + covar_file);
    // categorical covariates -> K-1 indicator columns (check_categories + get_dummies, src/Pheno.cpp:985-1010, :720-790);
    // any full-rank coding spans the same space, and only the column space of the covariates enters the analysis
    if (!ph.cat_cols.empty()) {
      std::vector<std::string> nn;
      std::vector<double> ee;
      for (size_t c = 0; c < cnames.size(); ++c) {
        if (!ph.cat_cols.count(cnames[c])) {
          nn.push_back(cnames[c]);
          ee.insert(ee.end(), cov.begin() + c * N, cov.begin() + (c + 1) * N);
          continue;
        }
        const int L = (int)levels[c].size();
        if (L > ph.max_cat_levels)
          throw Fail("too many categories for covariate: " + cnames[c] + " (=" + std::to_string(L) + "). Either use '--maxCatLevels' or combine categories.");
        if (L == 1) log << "WARNING: covariate ' " << cnames[c] << "' only has a single category so it will be ignored\n";
        for (int l = 1; l < L; ++l) {
          nn.push_back(cnames[c] + "_" + std::to_string(l));
          for (int64_t s = 0; s < N; ++s) {
            const double v = cov[c * N + s];
            ee.push_back(v == kMissing ? kMissing : (v == (double)l ? 1.0 : 0.0));
          }
        }
        if (L <= 1)                                            // keep missingness: a sample with NA here is still dropped
          for (int64_t s = 0; s < N; ++s) if (cov[c * N + s] == kMissing) in_cov[s] = 0;
      }
      cnames = nn;
      cov = ee;
    }
    log << " * covariates          : [" << covar_file << "] n_cov = " << cnames.size() << "\n";
    for (int64_t s = 0; s < N; ++s)
      for (size_t c = 0; c < cnames.size(); ++c)
        if (cov[c * N + s] == kMissing) in_cov[s] = 0;
  }
  ph.C = 1 + (int)cnames.size();
  ph.X.assign((size_t)N * ph.C, 0.0);
  for (int64_t s = 0; s < N; ++s) {
    ph.X[s] = 1.0;
    for (size_t c = 0; c < cnames.size(); ++c) ph.X[(c + 1) * N + s] = cov[c * N + s];
  }
  ph.in_analysis.assign(N, 0);
  for (int64_t s = 0; s < N; ++s) ph.in_analysis[s] = in_ph[s] && in_cov[s];
  ph.in_cov = in_cov;
}

// cyclic Jacobi eigen-decomposition of a small symmetric matrix (a: n x n row-major, destroyed);
// eigenvalues ascending in d, eigenvectors in the columns of v.
static void jacobi_eig(std::vector<double>& a, int n, std::vector<double>& d, std::vector<double>& v) {
  v.assign((size_t)n * n, 0.0);
  for (int i = 0; i < n; ++i) v[(size_t)i * n + i] = 1.0;
  for (int sweep = 0; sweep < 100; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < n; ++i) for (int j = i + 1; j < n; ++j) off += a[(size_t)i * n + j] * a[(size_t)i * n + j];
    if (off < 1e-300) break;
    for (int p = 0; p < n; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = a[(size_t)p * n + q];
        if (std::fabs(apq) < 1e-300) continue;
        const double theta = (a[(size_t)q * n + q] - a[(size_t)p * n + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = a[(size_t)k * n + p], akq = a[(size_t)k * n + q];
          a[(size_t)k * n + p] = c * akp - s * akq;
          a[(size_t)k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = a[(size_t)p * n + k], aqk = a[(size_t)q * n + k];
          a[(size_t)p * n + k] = c * apk - s * aqk;
          a[(size_t)q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = v[(size_t)k * n + p], vkq = v[(size_t)k * n + q];
          v[(size_t)k * n + p] = c * vkp - s * vkq;
          v[(size_t)k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  d.resize(n);
  std::vector<int> ord(n);
  for (int i = 0; i < n; ++i) { d[i] = a[(size_t)i * n + i]; ord[i] = i; }
  std::sort(ord.begin(), ord.end(), [&](int x, int y) { return d[x] < d[y]; });
  std::vector<double> d2(n), v2((size_t)n * n);
  for (int j = 0; j < n; ++j) {
    d2[j] = d[ord[j]];
    for (int k = 0; k < n; ++k) v2[(size_t)k * n + j] = v[(size_t)k * n + ord[j]];
  }
  d = d2; v = v2;
}

void get_basis(const std::vector<double>& X, int64_t N, int C0, std::vector<double>& Xb, int& nz) {
  std::vector<double> xtx((size_t)C0 * C0, 0.0), d, v;
  for (int a = 0; a < C0; ++a)
    for (int b = a; b < C0; ++b) {
      double s = 0.0;
      for (int64_t i = 0; i < N; ++i) s += X[(size_t)a * N + i] * X[(size_t)b * N + i];
      xtx[(size_t)a * C0 + b] = xtx[(size_t)b * C0 + a] = s;
    }
  jacobi_eig(xtx, C0, d, v);
  nz = 0;
  for (int j = 0; j < C0; ++j) if (d[j] > d[C0 - 1] * 1e-15) ++nz;
  Xb.assign((size_t)N * nz, 0.0);
  for (int j = 0; j < nz; ++j) {
    const int col = C0 - nz + j;
    const double inv = 1.0 / std::sqrt(d[col]);
    for (int a = 0; a < C0; ++a) {
      const double w = v[(size_t)a * C0 + col] * inv;
      if (w == 0.0) continue;
      for (int64_t i = 0; i < N; ++i) Xb[(size_t)j * N + i] += X[(size_t)a * N + i] * w;
    }
  }
}

// standard normal quantile: Acklam's rational approximation refined by one Halley step on erfc (~1e-16)
static double qnorm(double p) {
  static const double a[] = {-3.969683028665376e+01, 2.209460984245205e+02, -2.759285104469687e+02, 1.383577518672690e+02,
                             -3.066479806614716e+01, 2.506628277459239e+00};
  static const double b[] = {-5.447609879822406e+01, 1.615858368580409e+02, -1.556989798598866e+02, 6.680131188771972e+01,
                             -1.328068155288572e+01};
  static const double c[] = {-7.784894002430293e-03, -3.223964580411365e-01, -2.400758277161838e+00, -2.549732539343734e+00,
                             4.374664141464968e+00, 2.938163982698783e+00};
  static const double d[] = {7.784695709041462e-03, 3.224671290700398e-01, 2.445134137142996e+00, 3.754408661907416e+00};
  double x;
  if (p < 0.02425) {
    const double q = std::sqrt(-2 * std::log(p));
    x = (((((c[0] * q + c[1]) * q + c[2]) * q + c[3]) * q + c[4]) * q + c[5]) / ((((d[0] * q + d[1]) * q + d[2]) * q + d[3]) * q + 1);
  } else if (p > 1 - 0.02425) {
    const double q = std::sqrt(-2 * std::log(1 - p));
    x = -(((((c[0] * q + c[1]) * q + c[2]) * q + c[3]) * q + c[4]) * q + c[5]) / ((((d[0] * q + d[1]) * q + d[2]) * q + d[3]) * q + 1);
  } else {
    const double q = p - 0.5, r = q * q;
    x = (((((a[0] * r + a[1]) * r + a[2]) * r + a[3]) * r + a[4]) * r + a[5]) * q /
        (((((b[0] * r + b[1]) * r + b[2]) * r + b[3]) * r + b[4]) * r + 1);
  }
  for (int it = 0; it < 2; ++it) {
    const double e = 0.5 * std::erfc(-x / std::sqrt(2.0)) - p;
    const double u = e * std::sqrt(2 * M_PI) * std::exp(x * x / 2);
    x = x - u / (1 + x * u / 2);
  }
  return x;
}

// rank-based inverse normal transform per phenotype (apply_rint / rint_pheno, src/Pheno.cpp:1937-2010):
// average ranks for ties, quantile((rank - 3/8) / (n - 2 * 3/8 + 1))
static void apply_rint(Pheno& ph) {
  const int64_t N = ph.N;
  for (int p = 0; p < ph.P; ++p) {
    std::vector<std::pair<double, int64_t>> v;
    for (int64_t s = 0; s < N; ++s) {
      const double y = ph.Y[(size_t)p * N + s];
      if (y != kMissing && ph.mask[(size_t)p * N + s]) v.emplace_back(y, s);
    }
    std::sort(v.begin(), v.end(), [](const std::pair<double, int64_t>& x, const std::pair<double, int64_t>& z) { return x.first < z.first; });
    const size_t n = v.size();
    const double kc = 3.0 / 8.0;
    for (size_t i = 0; i < n;) {
      size_t e = i + 1;
      while (e < n && v[e].first == v[i].first) ++e;
      const double rank = (double)(i + 1) + (double)(e - i - 1) / 2.0;
      const double q = qnorm((rank - kc) / ((double)n - 2 * kc + 1));
      for (size_t j = i; j < e; ++j) ph.Y[(size_t)p * N + v[j].second] = q;
      i = e;
    }
  }
}

// setMasks (src/Pheno.cpp:810-841)
static void set_masks(Pheno& ph) {
  const int64_t N = ph.N;
  const int P = ph.P;
  for (int64_t s = 0; s < N; ++s) {
    bool any = false, all = true;
    for (int p = 0; p < P; ++p) { const bool m = ph.mask[(size_t)p * N + s]; any |= m; all &= m; }
    ph.in_analysis[s] = ph.in_analysis[s] && (ph.strict ? all : any);
    for (int p = 0; p < P; ++p) {
      ph.mask[(size_t)p * N + s] = ph.mask[(size_t)p * N + s] && ph.in_analysis[s];
      if (!ph.in_analysis[s]) {
        ph.Y[(size_t)p * N + s] *= 0.0;
        if (ph.bt) ph.Y_raw[(size_t)p * N + s] *= 0.0;
      }
    }
    if (!ph.in_analysis[s]) for (int c = 0; c < ph.C; ++c) ph.X[(size_t)c * N + s] = 0.0;
  }
  ph.n_analyzed = 0;
  for (int64_t s = 0; s < N; ++s) ph.n_analyzed += ph.in_analysis[s];
  if (ph.n_analyzed < 1) throw Fail("sample size cannot be < 1.");
  ph.neff.assign(P, 0.0);
  for (int p = 0; p < P; ++p) for (int64_t s = 0; s < N; ++s) ph.neff[p] += ph.mask[(size_t)p * N + s];
}

void prep_run(Pheno& ph, const std::vector<uint8_t>* extra_mask, Log& log) {
  const int64_t N = ph.N;
  const int P = ph.P;
  set_masks(ph);                                             // read_pheno_and_cov, src/Pheno.cpp:102
  if (ph.rint) {                                             // src/Pheno.cpp:111-115
    log << "   -applying RINT to all phenotypes\n";
    apply_rint(ph);
  }
  // pheno_impute_miss, QT (src/Pheno.cpp:1916-1931); binary traits keep the raw 0/1 values in Step 2
  for (int p = 0; p < P && ph.bt && ph.step1; ++p) {         // binary traits in Step 1: mean over the masked-in samples
    double tot = 0.0, ns = 0.0;
    for (int64_t s = 0; s < N; ++s)
      if (ph.mask[(size_t)p * N + s]) { tot += ph.Y[(size_t)p * N + s]; ns += 1.0; }
    for (int64_t s = 0; s < N; ++s) {
      double& y = ph.Y[(size_t)p * N + s];
      y = ph.mask[(size_t)p * N + s] ? y : 0.0 * (tot / ns);
    }
  }
  for (int p = 0; p < P && !ph.bt; ++p) {
    double tot = 0.0; int64_t ns = 0;
    for (int64_t s = 0; s < N; ++s) {
      const double y = ph.Y[(size_t)p * N + s];
      if (y != kMissing) { tot += y; if (ph.in_analysis[s]) ++ns; }
    }
    for (int64_t s = 0; s < N; ++s) {
      double& y = ph.Y[(size_t)p * N + s];
      if (y == kMissing) y = tot / (double)ns;
      y *= ph.mask[(size_t)p * N + s];
    }
  }
  if (extra_mask) {                                          // blup_read, src/Pheno.cpp:1306
    for (size_t e = 0; e < ph.mask.size(); ++e) ph.mask[e] = ph.mask[e] && (*extra_mask)[e];
    set_masks(ph);                                           // prep_run, src/Pheno.cpp:1070
  }
  log << " * number of individuals used in analysis = " << ph.n_analyzed << "\n";
  std::vector<double> Xb;
  int nz = 0;
  get_basis(ph.X, N, ph.C, Xb, nz);                           // getBasis (src/Pheno.cpp:1660-1681)
  ph.X = Xb;
  ph.C = nz;
  // residualize_phenotypes (src/Pheno.cpp:1813-1829)
  ph.scale_Y.assign(P, 1.0);
  for (int p = 0; p < P && (!ph.bt || ph.step1); ++p) {
    std::vector<double> beta(nz, 0.0);
    for (int c = 0; c < nz; ++c)
      for (int64_t i = 0; i < N; ++i) beta[c] += ph.Y[(size_t)p * N + i] * ph.X[(size_t)c * N + i];
    double ss = 0.0;
    for (int64_t i = 0; i < N; ++i) {
      double f = 0.0;
      for (int c = 0; c < nz; ++c) f += ph.X[(size_t)c * N + i] * beta[c];
      double& y = ph.Y[(size_t)p * N + i];
      y -= f * ph.mask[(size_t)p * N + i];
      ss += y * y;
    }
    ph.scale_Y[p] = std::sqrt(ss) / std::sqrt(ph.neff[p] - nz);
    if (ph.scale_Y[p] < 1e-6) throw Fail("phenotype '" + ph.names[p] + "' has sd=0.");
    for (int64_t i = 0; i < N; ++i) ph.Y[(size_t)p * N + i] /= ph.scale_Y[p];
  }
}

std::vector<Block> set_blocks(const std::vector<Snp>& snps, int bsize) {
  std::vector<Block> out;
  size_t i = 0;
  while (i < snps.size()) {
    size_t j = i;
    while (j < snps.size() && snps[j].chrom == snps[i].chrom) ++j;
    const size_t n = j - i;
    const size_t nb = (n + bsize - 1) / bsize;
    for (size_t b = 0; b < nb; ++b) {
      const size_t sz = ((b + 1) * bsize > n) ? n - b * bsize : (size_t)bsize;   // get_block_size :579-586
      out.push_back({snps[i].chrom, i + b * bsize, (int)sz});
    }
    i = j;
  }
  return out;
}

std::vector<int64_t> set_folds(const std::vector<uint8_t>& in_analysis, int k) {
  const int64_t n = (int64_t)in_analysis.size();
  int64_t na = 0;
  for (auto a : in_analysis) na += a;
  const int64_t target = na / k;
  if (target < 1) throw Fail("not enough samples are present for " + std::to_string(k) + "-fold CV.");
  std::vector<int64_t> sizes(k, 1);
  int64_t non_miss = 0, cum = 0;
  int cur = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (in_analysis[i]) ++non_miss;
    if (non_miss == target && cur < k - 1) {      // the last fold always takes the remainder (k < n_analyzed < 2k would overrun)
      sizes[cur] = i - cum + 1;
      cum += sizes[cur];
      non_miss = 0;
      ++cur;
    } else if (cur == k - 1) {
      sizes[cur] = n - i;
      break;
    }
  }
  return sizes;
}

std::vector<double> ridge_grid(int n) {
  if (n < 2) throw Fail("number of ridge parameters must be at least 2");
  std::vector<double> v(n);
  for (int i = 0; i < n; ++i) v[i] = (double)i / (n - 1);
  v[0] = 0.01;
  v[n - 1] = 0.99;
  return v;
}

}  // namespace rgh
