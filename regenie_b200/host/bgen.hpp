// BGEN v1.2 reader of the rgb200 host driver (layout 2, zlib / zstd / uncompressed, 8-bit, unphased, biallelic,
// diploid - the subset the reference's hand parser handles, src/Geno.cpp:2122-2345).  The file header and the
// variant identifying blocks (which the reference reads through the BGEN library, src/Geno.cpp:38-178) follow
// the public BGEN v1.2 specification; a bgenix index (<file>.bgi, SQLite) supplies the variant positions when present
// (read_bgi_file, src/Geno.cpp:180-309).  The inflated probability bytes go to the GPU unchanged.
#pragma once
#include "data.hpp"

namespace rgh {

struct BgenFile {
  std::string path;
  int sex_specific = 0;                        // 1 = males only, 2 = females only (set before open)
  std::vector<Snp> snps;                       // after --extract/--exclude; offset = file offset of the genotype block
  std::vector<std::string> keys_file, keys;
  std::vector<std::pair<std::string, std::string>> ids_file;   // (FID, IID) from --sample; empty for embedded ids
  std::vector<int> sex_file;                   // 1 = male, 2 = female, 0 = unknown (from --sample, else all 0)
  std::vector<int32_t> sample_idx;
  std::map<std::string, uint32_t> key_to_ind;
  uint32_t n_file = 0, n_variants_file = 0;
  int compression = 0;
  const uint8_t* data = nullptr;               // mmap of the whole file
  size_t size = 0;
  int fd = -1;
  ~BgenFile();
  void open(const std::string& path, const std::string& sample_file, bool ref_first, const std::set<std::string>& exclude,
            const std::set<std::string>& extract, const std::set<std::string>& remove, const std::set<std::string>& keep,
            const std::set<int>& chrs = {}, const std::string& bgi_file = "", bool no_bgi = false);
  bool used_bgi = false;                       // the variant positions came from <file>.bgi (or --bgi)
  // inflate variants snps[first .. first+n): probs [n][n_file][2], ploidy_missing [n][n_file]
  void read_block(size_t first, size_t n, uint8_t* probs, uint8_t* ploidy_missing, int threads) const;
  // variant-level imputation INFO over the analysed samples (info1 of compute_aaf_info, src/Geno.cpp:3134-3137, which
  // --minINFO compares against before any trait is looked at, :2074): 1 - sum(4 p_AA + p_het - g^2) / (2 n af (1 - af)),
  // from the inflated bytes of `n` variants; in_analysis is indexed like sample_idx (kept samples)
  void info_all(const uint8_t* probs, const uint8_t* ploidy_missing, size_t n, const uint8_t* in_analysis, bool ref_first,
                double* info_out, int threads) const;
  // the zlib streams of variants snps[first .. first+n) back to back, for rg_bgen_inflate (compression flag 1 only):
  // comp = concatenated streams, offs [n + 1]; throws when a variant's declared length is not 10 + 3 n_file
  void read_block_compressed(size_t first, size_t n, std::vector<uint8_t>& comp, std::vector<uint64_t>& offs) const;
};

}  // namespace rgh
