// Readers and phenotype/covariate preparation of the rgb200 host driver.
// Mirrors (restated, not copied) the reference's Geno/Pheno host logic:
//   read_bim src/Geno.cpp:518-611, read_fam :643-691, prep_bed :735-752,
//   pheno_read src/Pheno.cpp:148-364, covariate_read :573-700, setMasks :810-841,
//   pheno_impute_miss :1903-1935, getBasis :1660-1681, residualize_phenotypes :1799-1834,
//   set_blocks src/Data.cpp:311-334, set_folds :401-431.
#pragma once
#include <memory>
#include <set>

#include "util.hpp"

namespace rgh {

struct Snp {
  int chrom;
  std::string id;
  uint64_t pos;
  std::string allele0, allele1;   // ALLELE0 (reference), ALLELE1 (effect)
  uint64_t offset;                // row in the .bed / file offset of the genotype block in the .bgen
};

// the samples of the genotype file after --keep/--remove (params.FID_IID_to_ind)
struct SampleSet {
  const std::vector<std::string>& keys;
  const std::map<std::string, uint32_t>& key_to_ind;
};

struct PgenFile;

struct BedFile {
  std::string prefix;
  int sex_specific = 0;                       // 1 = males only, 2 = females only (set before open)
  std::shared_ptr<PgenFile> pg;               // set by open_pgen: rows are decoded from a .pgen into the same 2-bit layout
  std::vector<Snp> snps;                      // after --extract/--exclude
  std::vector<std::string> keys_file;         // FID_IID in .fam order
  std::vector<std::pair<std::string, std::string>> ids_file;   // (FID, IID) in .fam order (--write-samples)
  std::vector<int> sex_file;
  std::vector<std::string> keys;              // after --keep/--remove
  std::vector<int32_t> sample_idx;            // index in the .bed row of each kept sample
  std::map<std::string, uint32_t> key_to_ind; // FID_IID_to_ind
  uint64_t row_stride = 0;
  std::ifstream bed;
  int bed_fd = -1;                            // the same file for pread(): positioned reads from several threads, no shared cursor
  BedFile() = default;
  BedFile(const BedFile&) = delete;
  BedFile& operator=(const BedFile&) = delete;
  ~BedFile();
  void open(const std::string& prefix, bool ref_first, const std::set<std::string>& exclude,
            const std::set<std::string>& extract, const std::set<std::string>& remove,
            const std::set<std::string>& keep, const std::set<int>& chrs = {});
  // .pgen/.pvar/.psam behind the same interface (host/pgen.cpp); kernels then see ref-last PLINK 1 rows
  void open_pgen(const std::string& prefix, const std::set<std::string>& exclude, const std::set<std::string>& extract,
                 const std::set<std::string>& remove, const std::set<std::string>& keep, const std::set<int>& chrs = {});
  // read the rows of snps[first .. first+n) into out (n * row_stride bytes)
  void read_rows(size_t first, size_t n, uint8_t* out);
};

std::set<std::string> read_id_list(const std::string& path, int ncols);

struct Pheno {
  std::vector<std::string> names;
  int64_t N = 0;
  int P = 0, C = 0;
  std::vector<double> Y;          // N x P column-major (residualised + scaled for QT)
  std::vector<uint8_t> mask;      // N x P column-major
  std::vector<double> X;          // N x C column-major, orthonormal basis
  std::vector<uint8_t> in_analysis;
  std::vector<uint8_t> in_cov;    // samples with complete covariates (ind_in_cov_and_geno, src/Pheno.cpp:53)
  std::vector<double> neff, scale_Y;
  int64_t n_analyzed = 0;
  bool strict = false;
  bool bt = false, step1 = false;
  bool rint = false;              // --apply-rint
  std::vector<double> Y_raw;      // N x P raw 0/1 values (binary traits)
  std::set<std::string> pheno_cols, covar_cols;   // --phenoCol[List] / --covarCol[List] (empty = every column)
  std::set<std::string> pheno_excl, covar_excl;   // --phenoExcludeList / --covarExcludeList
  std::set<std::string> cat_cols;                 // --catCovarList: expanded to K-1 indicator columns
  int max_cat_levels = 10;                        // --maxCatLevels
  int min_case_count = 10;                        // --minCaseCount (binary traits)
};

// read_pheno_and_cov: raw values + masks, before prep_run
void read_pheno_and_cov(const SampleSet& g, const std::string& pheno_file, const std::string& covar_file,
                        bool step2, bool strict, bool bt, Pheno& ph, Log& log);
// orthonormal basis of the columns of X [C0][N] (getBasis, src/Pheno.cpp:1660-1681)
void get_basis(const std::vector<double>& X, int64_t N, int C0, std::vector<double>& Xb, int& nz);
// setMasks + orthonormal basis + residualise/scale (prep_run); `extra_mask` = LOCO availability (step 2)
void prep_run(Pheno& ph, const std::vector<uint8_t>* extra_mask, Log& log);

struct Block {
  int chrom;
  size_t first;
  int size;
};
std::vector<Block> set_blocks(const std::vector<Snp>& snps, int bsize);
std::vector<int64_t> set_folds(const std::vector<uint8_t>& in_analysis, int k);
std::vector<double> ridge_grid(int n);

}  // namespace rgh
