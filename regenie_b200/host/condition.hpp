// Conditional analysis (--condition-list [--condition-file FORMAT,FILE] [--max-condition-vars N]) of the rgb200 host
// driver.  Restated, not copied, from the reference:
//   get_conditional_vars src/Geno.cpp:4151-4179, get_snps_offset :4181-4215, extract_from_genofile :4217-4280,
//   setup_bed / setup_pgen / setup_bgen and read_snps_* :4282-4660, read_snp :3978-3996,
//   extract_condition_snps src/Pheno.cpp:952-983.
// The listed variants become extra covariate columns, appended after those of the covariate file and before the
// orthonormal basis is formed (getBasis); nothing downstream of the basis changes, so every GPU route conditions on
// them through the X matrix it already takes.  The IDs are also excluded from the tested variants and the Step-1 blocks.
#pragma once
#include <memory>

#include "bgen.hpp"
#include "data.hpp"

namespace rgh {

// columns the library accepts in X (kMaxCov of csrc/kernels.cuh): the basis of intercept + covariates + conditioning
// variants must fit, so a conditioned run that asks for more stops on the host before any GPU work
constexpr int kMaxCovColumns = 64;

struct Conditioning {
  std::string list_file;                      // --condition-list
  std::string fmt, file, sample_file;         // --condition-file FORMAT,FILE and --condition-file-sample (fmt empty: the main file)
  uint32_t max_vars = 10000;                  // --max-condition-vars
  bool ref_first = false;
  std::set<std::string> ids;                  // the listed IDs, in the ID order of the reference's std::map

  bool on() const { return !list_file.empty(); }
  bool external() const { return !fmt.empty(); }
  // reads the list (get_conditional_vars); the IDs then go into the exclusion set of the main reader
  void read_list();
  // same-file conditioning: finds the IDs in the main genotype file (format "bed" / "pgen" / "bgen") among the variants
  // of the --chr / --range selection, before --extract / --exclude (check_snps_include_exclude, src/Geno.cpp:1136-1137)
  void locate_in_main(const std::string& main_fmt, const std::string& path, const std::string& sample, const std::string& bgi,
                      const std::set<int>& chrs, bool set_range, int range_chr, double range_min, double range_max);
  // appends the conditioning columns to ph.X (after read_pheno_and_cov, before prep_run): the genotype of each variant
  // over the samples of `g`, missing calls and samples absent from the file set to the mean over ph.in_cov
  void append(const SampleSet& g, Pheno& ph, Log& log);

 private:
  std::string src_fmt;
  std::unique_ptr<BedFile> bed;               // .bed or .pgen (2-bit rows)
  std::unique_ptr<BgenFile> bgen;
  std::vector<size_t> rows;                   // per ID (in `ids` order): index into the source reader's snps
  void open_source(const std::string& f, const std::string& path, const std::string& sample, const std::string& bgi,
                   const std::set<int>& chrs);
  void find(bool same_file, bool set_range, int range_chr, double range_min, double range_max);
};

}  // namespace rgh
