// rgb200 -- host driver keeping regenie's CLI surface for the Step-1 / Step-2 hot path and calling
// the sm_90a kernels through the C ABI (include/rg_b200.h).
// Mirrors the control flow of the reference driver (restated, not copied):
//   main / read_params_and_check   src/Regenie.cpp:60-142
//   Data::run_step1                src/Data.cpp:95-133   (level_0_calculations :594, output :956,
//                                                         write_predictions :1795)
//   Data::test_snps_fast           src/Data.cpp:2230-2383 (compute_res :2386, printing
//                                                         src/Step2_Models.cpp:2386-2540)
#include <algorithm>
#include <chrono>
#include <cstring>
#include <climits>
#include <cstdlib>
#include <future>
#include <iomanip>
#include <limits>

#include "../../include/rg_b200.h"
#include <mutex>
#include <thread>

#include "bgen.hpp"
#include "bt_null.hpp"
#include "data.hpp"
#include "output.hpp"
#include "pgen.hpp"

#include <unistd.h>

using namespace rgh;

namespace {

struct Params {
  int step = 0;
  std::string bed, bgen, pgen, sample, pheno, covar, out, pred, lowmem_prefix;
  std::string remove, keep, exclude, extract;
  int bsize = 0, cv = 5, l0 = 5, l1 = 5, gpu = 0;
  bool loocv = false, lowmem = false, ref_first = false, strict = false, bt = false, force_step1 = false;
  bool rel_path = false, firth = false, approx = false, keep_l0 = false, spa = false;
  double min_mac = 5.0, p_thresh = 0.05;
  int threads = 0;
  std::set<int> chrs;                 // --chr / --chrList
  std::set<std::string> pheno_cols, covar_cols;   // --phenoCol / --phenoColList / --covarCol / --covarColList
  double min_info = 0.0;                       // --minINFO (dosage input)
  bool ignore_pred = false;                    // --ignore-pred: Step 2 without the LOCO offsets
  bool rint = false;                           // --apply-rint
  std::set<std::string> cat_cols;              // --catCovarList
  int max_cat_levels = 10;                     // --maxCatLevels
  std::string split_prefix, master;   // --split-l0 PREFIX,N / --run-l0 FILE,K / --run-l1 FILE
  int split_jobs = 0, run_l0_job = 0;
  bool run_l1 = false;
  bool gz = false;                             // --gz: .loco / .prs / .regenie outputs through zlib (file names gain ".gz")
  bool write_samples = false, print_pheno = false;   // --write-samples [--print-pheno]: <out>_<pheno>.regenie.ids
  bool print_prs = false, use_prs = false;     // --print-prs (step 1) / --use-prs (step 2)
  std::string bgi;                             // --bgi FILE (default: <bgen>.bgi when it exists)
  std::vector<double> setl0, setl1;            // --setl0 / --setl1: user ridge grids in (0,1)
  std::set<std::string> pheno_excl, covar_excl, l1_phenos;   // --phenoExcludeList / --covarExcludeList / --l1-phenoList
  bool set_range = false;                      // --range CHR:MINPOS-MAXPOS (step 2)
  int range_chr = 0;
  double range_min = 0, range_max = 0;
  bool write_null_firth = false;               // --write-null-firth (step 1, binary traits)
  std::string null_firth_list;                 // --use-null-firth FILE (step 2)
  int sex_specific = 0;                        // --sex-specific male|female
  int start_block = 1;                         // --starting-block (step 2)
  bool af_cc = false;                          // --af-cc: A1FREQ / N among cases and controls (binary traits, split output)
  int min_case_count = 10;                     // --minCaseCount
  bool no_split = false;                       // --no-split: one <out>.regenie for all traits (hard-call input)
  std::string htp_cohort;                      // --htp COHORT: HTPv4 rows (src/Step2_Models.cpp:2400-2426, :2542-2646); autosomes
  bool htp = false;
  int test_type = 0;                           // --test additive | dominant | recessive (step 2)
  int gpus = 1;                                // --gpus N (step 1): level-0 blocks sharded over N GPUs of this node, level 1 by phenotype
  bool gpu_inflate = false;                    // --gpu-inflate: zlib payloads of the .bgen are inflated on the device (rg_bgen_inflate)
  uint32_t par1_max = 2781479, par2_min = 155701383;   // hg38 (check_build_code, src/Regenie.cpp:1643-1660)
};

void rg_check(int rc) {
  if (rc != 0) throw Fail(std::string(rg_last_error()));
}

// The driver is one run per process: when it is done, device buffers, pinned memory and the CUDA context go back with
// the process, so main() leaves through _exit once every output file is closed (freeing ~10 GB of device buffers one
// cudaFree at a time and tearing the context down costs more than level 0 of the benchmark panel).
// RG_B200_CLEAN_EXIT=1 runs every destructor instead (leak checkers, compute-sanitizer).
static const bool g_fast_exit = getenv("RG_B200_CLEAN_EXIT") == nullptr;

// releases a handle on every way out of a run function (errors unwind through here)
struct HandleGuard {
  rg_handle& h;
  ~HandleGuard() {
    if (h && !g_fast_exit) rg_destroy(h);
    h = nullptr;
  }
};

// get_unit_params (src/Regenie.cpp:1477-1495): sorted unique values strictly inside (0, 1)
std::vector<double> unit_params(const std::string& opt, const std::string& csv) {
  std::vector<double> v;
  std::string tok;
  std::istringstream ss(csv);
  while (std::getline(ss, tok, ',')) if (!tok.empty()) v.push_back(convert_double(tok));
  std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  for (double x : v) if (x <= 0 || x >= 1) throw Fail("must specify values for " + opt + " in (0,1).");
  if (v.empty()) throw Fail("must specify values for " + opt + " in (0,1).");
  return v;
}

// check_name (src/Regenie.cpp:1596-1645): "V{1:3}x" -> V1x, V2x, V3x
std::vector<std::string> expand_name(const std::string& str) {
  std::vector<std::string> out;
  if (str.empty()) return out;
  const size_t lb = str.find('{');
  if (lb == std::string::npos) { out.push_back(str); return out; }
  const std::string err = "invalid string expansion (=" + str + ").";
  const size_t colon = str.find(':'), rb = str.find('}');
  if (colon == std::string::npos || rb == std::string::npos || colon < lb || rb < colon) throw Fail(err);
  char* e1 = nullptr;
  char* e2 = nullptr;
  const std::string a = str.substr(lb + 1, colon - lb - 1), b = str.substr(colon + 1, rb - colon - 1);
  const long imin = strtol(a.c_str(), &e1, 10), imax = strtol(b.c_str(), &e2, 10);
  if (a.empty() || b.empty() || *e1 || *e2) throw Fail(err);
  for (long j = imin; j <= imax; ++j) out.push_back(str.substr(0, lb) + std::to_string(j) + str.substr(rb + 1));
  return out;
}

Params parse_cli(int argc, char** argv) {
  Params p;
  auto csv_into = [](const std::string& v, std::set<std::string>& dst) {
    std::string tok;
    std::istringstream ss(v);
    while (std::getline(ss, tok, ','))
      for (const auto& n : expand_name(tok)) dst.insert(n);
  };
  auto need = [&](int& i) -> std::string {
    if (i + 1 >= argc) throw Fail(std::string("option ") + argv[i] + " needs a value");
    return argv[++i];
  };
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--step") p.step = atoi(need(i).c_str());
    else if (a == "--version" || a == "-v") { std::cout << "rgb200 (" << rg_version() << ")\n"; exit(0); }
    else if (a == "--setl0") { p.setl0 = unit_params("--l0", need(i)); p.l0 = (int)p.setl0.size(); }
    else if (a == "--setl1") { p.setl1 = unit_params("--l1", need(i)); p.l1 = (int)p.setl1.size(); }
    else if (a == "--phenoExcludeList") csv_into(need(i), p.pheno_excl);
    else if (a == "--covarExcludeList") csv_into(need(i), p.covar_excl);
    else if (a == "--l1-phenoList") csv_into(need(i), p.l1_phenos);
    else if (a == "--bed") p.bed = need(i);
    else if (a == "--bgen") p.bgen = need(i);
    else if (a == "--pgen") p.pgen = need(i);
    else if (a == "--phenoFile" || a == "-p") p.pheno = need(i);
    else if (a == "--covarFile" || a == "-c") p.covar = need(i);
    else if (a == "--bsize" || a == "-b") p.bsize = atoi(need(i).c_str());
    else if (a == "--out" || a == "-o") p.out = need(i);
    else if (a == "--pred") p.pred = need(i);
    else if (a == "--cv") p.cv = atoi(need(i).c_str());
    else if (a == "--l0") p.l0 = atoi(need(i).c_str());
    else if (a == "--l1") p.l1 = atoi(need(i).c_str());
    else if (a == "--remove") p.remove = need(i);
    else if (a == "--keep") p.keep = need(i);
    else if (a == "--exclude") p.exclude = need(i);
    else if (a == "--extract") p.extract = need(i);
    else if (a == "--minMAC") p.min_mac = atof(need(i).c_str());
    else if (a == "--lowmem-prefix") p.lowmem_prefix = need(i);
    else if (a == "--gpu") p.gpu = atoi(need(i).c_str());
    else if (a == "--gpus") p.gpus = atoi(need(i).c_str());
    else if (a == "--threads") p.threads = atoi(need(i).c_str());   // host threads: BGEN inflate only
    else if (a == "--sample") p.sample = need(i);
    else if (a == "--phenoCol") csv_into(need(i), p.pheno_cols);
    else if (a == "--covarCol") csv_into(need(i), p.covar_cols);
    else if (a == "--phenoColList") csv_into(need(i), p.pheno_cols);
    else if (a == "--covarColList") csv_into(need(i), p.covar_cols);
    else if (a == "--minINFO") p.min_info = atof(need(i).c_str());
    else if (a == "--ignore-pred") p.ignore_pred = true;
    else if (a == "--apply-rint") p.rint = true;
    else if (a == "--catCovarList") csv_into(need(i), p.cat_cols);
    else if (a == "--maxCatLevels") p.max_cat_levels = atoi(need(i).c_str());
    else if (a == "--split-l0" || a == "--run-l0") {
      const std::string v = need(i);
      const size_t k = v.find_last_of(',');
      if (k == std::string::npos || atoi(v.c_str() + k + 1) < 1)
        throw Fail("wrong format for " + a + " (must be FILE,INT).");
      if (a == "--split-l0") { p.split_prefix = v.substr(0, k); p.split_jobs = atoi(v.c_str() + k + 1); }
      else { p.master = v.substr(0, k); p.run_l0_job = atoi(v.c_str() + k + 1); }
    }
    else if (a == "--run-l1") { p.master = need(i); p.run_l1 = true; }
    else if (a == "--par-region") {
      const std::string v = need(i);
      int lo = 0, hi = 0;
      if (v == "b36" || v == "hg18") { p.par1_max = 2709520; p.par2_min = 154584238; }
      else if (v == "b37" || v == "hg19") { p.par1_max = 2699520; p.par2_min = 154931044; }
      else if (v == "b38" || v == "hg38") { p.par1_max = 2781479; p.par2_min = 155701383; }
      else if (sscanf(v.c_str(), "%d,%d", &lo, &hi) == 2 && lo >= 1 && hi >= lo) { p.par1_max = lo - 1; p.par2_min = hi + 1; }
      else throw Fail("invalid build code given (valid ones are 'b36|b37|b38|hg18|hg19|hg38' or [start,end] position of the non-par region)");
    }
    else if (a == "--chr") { const int c = chr_str_to_int(need(i)); if (c < 1) throw Fail("invalid chromosome for --chr."); p.chrs.insert(c); }
    else if (a == "--chrList") {
      std::string v = need(i), tok;
      std::istringstream ss(v);
      while (std::getline(ss, tok, ',')) { const int c = chr_str_to_int(tok); if (c < 1) throw Fail("invalid chromosome in --chrList."); p.chrs.insert(c); }
    }
    else if (a == "--pThresh") p.p_thresh = atof(need(i).c_str());
    else if (a == "--firth") p.firth = true;
    else if (a == "--approx") p.approx = true;
    else if (a == "--spa") p.spa = true;
    else if (a == "--loocv") p.loocv = true;
    else if (a == "--lowmem") p.lowmem = true;     // W stays resident in HBM; files only with --keep-l0
    else if (a == "--keep-l0") p.keep_l0 = true;
    else if (a == "--ref-first") p.ref_first = true;
    else if (a == "--strict") p.strict = true;
    else if (a == "--qt" || a == "--force-qt") {}   // QT is the default; 0/1 phenotypes are taken as they are
    else if (a == "--gz") p.gz = true;
    else if (a == "--write-samples") p.write_samples = true;
    else if (a == "--print-pheno") p.print_pheno = true;
    else if (a == "--print-prs") p.print_prs = true;
    else if (a == "--use-prs") p.use_prs = true;
    else if (a == "--bgi") p.bgi = need(i);
    else if (a == "--gpu-inflate") p.gpu_inflate = true;
    else if (a == "--no-split") p.no_split = true;
    else if (a == "--htp") { p.htp_cohort = need(i); p.htp = true; }
    else if (a == "--af-cc") p.af_cc = true;
    else if (a == "--sex-specific") {                          // src/Regenie.cpp:756-762
      const std::string v = need(i);
      if (v == "male") p.sex_specific = 1;
      else if (v == "female") p.sex_specific = 2;
      else throw Fail("unrecognized argument for option --sex-specific, must be either 'male' or 'female'.");
    }
    else if (a == "--starting-block") p.start_block = atoi(need(i).c_str());
    else if (a == "--write-null-firth") p.write_null_firth = true;
    else if (a == "--use-null-firth") p.null_firth_list = need(i);
    else if (a == "--minCaseCount") p.min_case_count = atoi(need(i).c_str());
    else if (a == "--test") {                                   // src/Regenie.cpp:735-740
      const std::string v = need(i);
      if (v == "additive") p.test_type = 0;
      else if (v == "dominant") p.test_type = 1;
      else if (v == "recessive") p.test_type = 2;
      else throw Fail("unrecognized argument for option --test, must be either 'additive', 'dominant' or 'recessive'.");
    }
    else if (a == "--range") {                                  // src/Regenie.cpp:741-755
      char chr[20];
      double p0 = -1, p1 = -1;
      const std::string v = need(i);
      if (sscanf(v.c_str(), "%19[^:]:%lf-%lf", chr, &p0, &p1) != 3 || p0 < 0 || p1 < 0)
        throw Fail("wrong format for --range (must be CHR:MINPOS-MAXPOS).");
      p.range_chr = chr_str_to_int(chr);
      p.range_min = std::min(p0, p1);
      p.range_max = std::max(p0, p1);
      p.set_range = true;
    }
    else if (a == "--bt") p.bt = true;
    else if (a == "--force-step1") p.force_step1 = true;
    else if (a == "--use-relative-path") p.rel_path = true;
    else if (a == "--help" || a == "-h") {
      std::cout << "rgb200: H100-native regenie Step 1 / Step 2 hot path\n"
                   "  --step 1|2 --bed PREFIX | --pgen PREFIX | --bgen FILE --phenoFile F [--covarFile F] --bsize N --out PREFIX\n"
                   "  [--pred LIST] [--loocv] [--lowmem] [--cv K] [--l0 R] [--l1 R] [--remove F] [--keep F]\n"
                   "  [--exclude F] [--extract F] [--ref-first] [--minMAC x] [--strict] [--gpu ordinal]\n"
                   "  [--phenoCol c]... [--phenoColList a,b] [--covarCol c]... [--covarColList a,b] [--minINFO x] [--ignore-pred]\n"
                   "  [--chr c]... [--chrList c1,c2,...] [--range CHR:MIN-MAX]  (Step-2 jobs are split by chromosome / window like the reference)\n"
                   "  step 2 binary traits: --bt [--firth --approx | --spa] [--pThresh p] with --bed or --bgen F [--sample F] [--bgi F]\n"
                   "  [--gz] [--print-prs | --use-prs] [--write-samples [--print-pheno]]  (.gz inputs are read by file name)\n"
                   "  [--test additive|dominant|recessive] [--no-split] [--af-cc] [--minCaseCount n] [--write-null-firth | --use-null-firth F]\n"
                   "  [--gpus N]  step 1: shard the level-0 blocks over N GPUs of this node (level 1 by phenotype), same output files\n"
                   "  [--gpu-inflate]  step 2 on zlib-compressed .bgen: inflate the genotype blocks on the GPU instead of the host\n";
      exit(0);
    } else {
      throw Fail("option '" + a + "' is outside the hot path covered by rgb200 (see DESIGN.md, out of scope)");
    }
  }
  if (!p.setl0.empty()) p.l0 = (int)p.setl0.size();
  if (!p.setl1.empty()) p.l1 = (int)p.setl1.size();
  if (p.step != 1 && p.step != 2) throw Fail("specify which mode regenie should be running using option '--step'.");
  if ((!p.bgen.empty()) + (!p.bed.empty()) + (!p.pgen.empty()) > 1) throw Fail("specify only one genotype input (--bed, --pgen or --bgen).");
  if (!p.pgen.empty()) p.ref_first = false;          // .pgen rows are emitted as ref-last PLINK 1 rows counting ALT
  if (p.firth && p.spa) throw Fail("cannot use both --firth and --spa.");
  if (p.firth && !p.approx) throw Fail("exact Firth (--firth without --approx) is outside the hot path covered by rgb200; use --firth --approx.");
  if (p.bed.empty() && p.bgen.empty() && p.pgen.empty()) throw Fail("must specify the genotype file with --bed, --pgen or --bgen.");
  if (p.pheno.empty()) throw Fail("must provide the phenotype file with --phenoFile.");
  if ((p.split_jobs || p.run_l0_job || p.run_l1) && p.step != 1) throw Fail("options --split-l0/--run-l0/--run-l1 only work in step 1.");
  if (p.out.empty()) throw Fail("must specify an output file prefix with --out.");
  if (p.bsize < 1) throw Fail("must specify the block size using '--bsize'.");
  if (p.test_type > 0 && p.step != 2) throw Fail("can only use --test in step 2 (association testing).");   // src/Regenie.cpp:905-906
  if (p.set_range && p.range_chr == -1) throw Fail("unrecognized chromosome in --range.");   // src/Regenie.cpp:1153-1154
  if (p.write_samples && !p.bgen.empty() && p.sample.empty())                     // src/Regenie.cpp:903-904
    throw Fail("must specify sample file (using --sample) if writing sample IDs to file.");
  if (p.step == 2 && p.pred.empty() && !p.ignore_pred) throw Fail("must specify --pred if using --step 2 (otherwise use --ignore-pred).");
  if (p.htp) {
    if (p.step != 2) throw Fail("option --htp only works in step 2.");
    if (p.no_split) p.no_split = false;                       // src/Regenie.cpp:1068-1071: --no-split is ignored with --htp
  }
  return p;
}

std::string full_path(const std::string& f, bool rel) {
  if (rel) return f;
  char buf[PATH_MAX];
  if (realpath(f.c_str(), buf)) return std::string(buf);
  // file may not exist yet: resolve the directory part
  const size_t k = f.find_last_of('/');
  const std::string dir = (k == std::string::npos) ? "." : f.substr(0, k);
  const std::string base = (k == std::string::npos) ? f : f.substr(k + 1);
  if (realpath(dir.c_str(), buf)) return std::string(buf) + "/" + base;
  return f;
}

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

// RG_B200_PHASES=1: wall-clock of the driver's phases on stderr (bench.py's from-files leg reads them); no effect on outputs
static void phase(const char* name) {
  static const bool on = getenv("RG_B200_PHASES") != nullptr;
  static const double t_start = now_ms();
  static double t_last = t_start;
  if (!on) return;
  const double t = now_ms();
  fprintf(stderr, "[phase] %-22s %9.1f ms  (+%.1f)\n", name, t - t_start, t - t_last);
  t_last = t;
}

static std::shared_future<int> g_ndev;              // number of CUDA devices, from the warm-up thread started in main()
static void require_device() {
  if (g_ndev.valid() && g_ndev.get() < 1) throw Fail("no CUDA device available: rgb200 has no CPU fallback");
}

// ------------------------------------------------------------------------------------ step 1
// .pgen input: the records of a block go to the GPU as they are and are expanded there (rg_pgen_decode, SURVEY 8 (f)3).
// RG_B200_PGEN=host selects the host decoder (host/pgen.cpp), which also serves the options that edit rows on the host
// (--no-split genotype counts, --test dominant / recessive, --af-cc).
static bool pgen_on_device() {
  const char* e = getenv("RG_B200_PGEN");
  return !(e && std::string(e) == "host");
}
static void pgen_rows_device(rg_handle h, const PgenBatch& pb, int bs, int64_t n_file, int block_id, const uint8_t** rows,
                             int64_t* stride) {
  rg_pgen_block blk{pb.bytes.data(), (int64_t)pb.bytes.size(), pb.rec_off.data(), pb.rec_len.data(), pb.rec_type.data(),
                    (int32_t)pb.rec_off.size(), pb.own.data(), pb.base.data(), bs, n_file, block_id};
  rg_check(rg_pgen_decode(h, &blk, rows, stride));
}

// .bed/.bim/.fam or .pgen/.pvar/.psam behind the same row interface
void open_rows(const Params& p, BedFile& g, const std::set<std::string>& excl, const std::set<std::string>& extr,
               const std::set<std::string>& rem, const std::set<std::string>& keep, Log& log) {
  g.sex_specific = p.sex_specific;
  if (p.sex_specific) log << "   -keeping only " << (p.sex_specific == 1 ? "male" : "female") << " individuals in the analysis\n";
  if (!p.pgen.empty()) {
    g.open_pgen(p.pgen, excl, extr, rem, keep, p.chrs);
    log << " * pvar                : [" << p.pgen << ".pvar] n_snps = " << g.snps.size() << "\n";
    log << " * psam                : [" << p.pgen << ".psam] n_samples = " << g.keys.size() << "\n";
  } else {
    g.open(p.bed, p.ref_first, excl, extr, rem, keep, p.chrs);
    log << " * bim                 : [" << p.bed << ".bim] n_snps = " << g.snps.size() << "\n";
    log << " * fam                 : [" << p.bed << ".fam] n_samples = " << g.keys.size() << "\n";
  }
}

// ---- --split-l0 / --run-l0 / --run-l1 (src/Data.cpp:232-309, 818-908): level 0 as independent jobs that exchange
// the N x R slabs of write_l0_file through <prefix>_job<j>_l0_Y<k>; files are interchangeable with the reference's.
struct MasterJob { std::string prefix; int nblocks; long nsnps; };
struct Master { long n_geno = 0; int bsize = 0; std::vector<MasterJob> jobs; };

Master read_master(const std::string& path, int bsize) {
  std::ifstream fh(path);
  if (!fh) throw Fail("cannot open file : " + path);
  Master m;
  std::string line;
  if (!std::getline(fh, line)) throw Fail("cannot read header line in master file.");
  if (sscanf(line.c_str(), "%ld %d", &m.n_geno, &m.bsize) != 2 || m.bsize != bsize) throw Fail("invalid header line in master file.");
  while (std::getline(fh, line)) {
    auto t = split_ws(line);
    if (t.empty()) continue;
    if (t.size() != 3) throw Fail("could not read line " + std::to_string(m.jobs.size() + 2) + " (check number of lines and format in file).");
    m.jobs.push_back({t[0], atoi(t[1].c_str()), atol(t[2].c_str())});
  }
  return m;
}

void write_master(const Params& p, const std::vector<Snp>& snps, const std::vector<Block>& blocks, Log& log) {
  int njobs = p.split_jobs;
  const int nb_tot = (int)blocks.size();
  log << " * running level 0 in parallel across " << nb_tot << " genotype blocks\n";
  if (njobs <= 1) throw Fail("number of jobs must be >1.");
  if (njobs > nb_tot) { log << "   -WARNING: Number of jobs cannot be greater than number of blocks.\n"; njobs = nb_tot; }
  const std::string fout = p.split_prefix + ".master";
  log << "   -using " << njobs << " jobs\n   -master file written to [" << fout << "]\n"
      << "   -variant list files written to [" << p.split_prefix << "_job*.snplist]\n";
  std::ofstream of(fout);
  if (!of) throw Fail("cannot write to file : " + fout);
  of << snps.size() << " " << p.bsize << "\n";
  const int nall = nb_tot / njobs, rem = nb_tot - nall * njobs;
  int b = 0;
  for (int j = 0; j < njobs; ++j) {
    const int target = nall + (j < rem ? 1 : 0);
    const std::string fname = p.split_prefix + "_job" + std::to_string(j + 1);
    long ns = 0;
    std::ofstream sl(fname + ".snplist");
    if (!sl) throw Fail("cannot write to file : " + fname + ".snplist");
    for (int k = 0; k < target; ++k, ++b) {
      for (int v = 0; v < blocks[b].size; ++v) sl << snps[blocks[b].first + v].id << "\n";
      ns += blocks[b].size;
    }
    of << fname << " " << target << " " << ns << "\n";
  }
}

void run_step1(const Params& p_in, Log& log) {
  Params p = p_in;
  if (p.af_cc) log << "WARNING: disabling option --af-cc (only for BTs in step 2 in native output format split by trait).\n";
  if (p.set_range) { log << "WARNING: option --range only works for step 2.\n"; p.set_range = false; }
  Master master;
  if (p.run_l0_job || p.run_l1) master = read_master(p.master, p.bsize);
  if (p.run_l0_job) {
    if (p.run_l0_job > (int)master.jobs.size()) throw Fail("could not read line " + std::to_string(p.run_l0_job + 1) + " (check number of lines in file).");
    log << " * running jobs in parallel (job #" << p.run_l0_job << ")\n";
    p.extract = master.jobs[p.run_l0_job - 1].prefix + ".snplist";       // file_snps_include (src/Data.cpp:852-854)
    p.exclude.clear();
    p.lowmem_prefix = master.jobs[p.run_l0_job - 1].prefix;
  }
  // genotype input: 2-bit rows (.bed / decoded .pgen) or 8-bit dosages (.bgen, readChunkFromBGENFileToG_fast src/Geno.cpp:1574)
  const bool use_bgen = !p.bgen.empty();
  BedFile gbed;
  BgenFile gg;
  if (use_bgen) {
    gg.open(p.bgen, p.sample, p.ref_first, read_id_list(p.exclude, 1), read_id_list(p.extract, 1), read_id_list(p.remove, 2),
            read_id_list(p.keep, 2), p.chrs, p.bgi);
    if (gg.used_bgi) log << "   -index bgi file [" << (p.bgi.empty() ? p.bgen + ".bgi" : p.bgi) << "]\n";
    log << " * bgen                : [" << p.bgen << "] n_snps = " << gg.snps.size() << ", n_samples = " << gg.keys.size() << "\n";
  } else {
    open_rows(p, gbed, read_id_list(p.exclude, 1), read_id_list(p.extract, 1), read_id_list(p.remove, 2), read_id_list(p.keep, 2), log);
  }
  // the fields of either reader the rest of Step 1 needs
  struct GenoView {
    const std::vector<Snp>& snps;
    const std::vector<std::string>& keys;
    const std::map<std::string, uint32_t>& key_to_ind;
    const std::vector<int32_t>& sample_idx;
    size_t n_file;
    size_t row_stride;
  };
  const GenoView g = use_bgen ? GenoView{gg.snps, gg.keys, gg.key_to_ind, gg.sample_idx, (size_t)gg.n_file, 0}
                              : GenoView{gbed.snps, gbed.keys, gbed.key_to_ind, gbed.sample_idx, gbed.keys_file.size(), (size_t)gbed.row_stride};
  if (g.snps.empty()) throw Fail("no variant left to include in analysis.");
  if (g.snps.size() > 1000000 && !p.force_step1)
    throw Fail("it is not recommened to use more than 1000000 variants in step 1 (otherwise use '--force-step1').");
  Pheno ph;
  ph.pheno_cols = p.pheno_cols; ph.covar_cols = p.covar_cols; ph.rint = p.rint && !p.bt; ph.cat_cols = p.cat_cols; ph.max_cat_levels = p.max_cat_levels;
  ph.pheno_excl = p.pheno_excl; ph.covar_excl = p.covar_excl; ph.min_case_count = p.min_case_count;
  read_pheno_and_cov(SampleSet{g.keys, g.key_to_ind}, p.pheno, p.covar, false, p.strict, p.bt, ph, log);
  prep_run(ph, nullptr, log);
  if (p.bt && !p.loocv) {
    if (ph.n_analyzed < 5000) {                       // src/Data.cpp:353-356
      log << "   -WARNING: Sample size is less than 5,000 so using LOOCV instead of " << p.cv << "-fold CV.\n";
      p.loocv = true;
    }
  }
  const auto blocks = set_blocks(g.snps, p.bsize);
  const int nb = (int)blocks.size();
  if (p.split_jobs) { write_master(p, g.snps, blocks, log); return; }
  if (p.run_l0_job) {
    const MasterJob& mj = master.jobs[p.run_l0_job - 1];
    if (mj.nblocks != nb || mj.nsnps != (long)g.snps.size())
      throw Fail("number of variants/blocks in file (=" + std::to_string(g.snps.size()) + "/" + std::to_string(nb) +
                 ") don't match with that in master file (=" + std::to_string(mj.nsnps) + "/" + std::to_string(mj.nblocks) + ").");
  }
  if (p.run_l1) {
    long tb = 0, ts = 0;
    for (auto& j : master.jobs) { tb += j.nblocks; ts += j.nsnps; }
    if (tb != nb || ts != (long)g.snps.size())
      throw Fail("number of blocks/variants in master file '" + p.master + "' doesn't match that in the analysis.");
    log << " * using results from running " << master.jobs.size() << " parallel jobs at level 0\n";
  }
  const int64_t N = ph.N;
  const int P = ph.P;
  std::vector<int64_t> folds;
  if (!p.loocv) folds = set_folds(ph.in_analysis, p.cv);
  if ((p.setl0.empty() && p.l0 < 2) || (p.setl1.empty() && p.l1 < 2))                 // set_ridge_params, src/Regenie.cpp:1499-1500
    throw Fail("number of ridge parameters must be at least 2 (=" + std::to_string(p.setl0.empty() && p.l0 < 2 ? p.l0 : p.l1) + ")");
  const auto h0 = p.setl0.empty() ? ridge_grid(p.l0) : p.setl0, h1 = p.setl1.empty() ? ridge_grid(p.l1) : p.setl1;
  std::vector<double> lambda(p.l0);
  const double M = p.run_l0_job ? (double)master.n_geno : (double)g.snps.size();     // src/Data.cpp:607
  for (int j = 0; j < p.l0; ++j) lambda[j] = M * (1 - h0[j]) / h0[j];           // src/Data.cpp:607
  log << " * # blocks            : [" << nb << "] for " << g.snps.size() << " variants\n";
  log << " * # CV folds          : [" << (p.loocv ? ph.n_analyzed : p.cv) << "]\n";

  rg_step1_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.device = p.gpu; cfg.n_samples = N; cfg.n_cov = ph.C; cfg.n_pheno = P; cfg.n_folds = p.cv;
  cfg.n_ridge_l0 = p.l0; cfg.n_ridge_l1 = p.l1; cfg.loocv = p.loocv; cfg.max_block_size = p.bsize;
  cfg.total_blocks = nb; cfg.n_analyzed = ph.n_analyzed;
  // --gpus G: one handle per device, all describing the same problem.  Level-0 blocks are partitioned contiguously by the
  // reference's --split-l0 rule (write_l0_master, src/Data.cpp:268-301), level 1 by phenotype (p mod G); every GPU stores the
  // predictor tiles of a phenotype straight into the HBM of the GPU that owns it (peer access over NVLink), so there is no
  // exchange step and no file protocol.  Results do not depend on G (fixed-order reductions).
  const int G = std::max(1, p.gpus);
  if (G > 1) {
    if (G > rg_device_count()) throw Fail("--gpus " + std::to_string(G) + " but only " + std::to_string(rg_device_count()) + " CUDA device(s) visible.");
    if (G > nb) throw Fail("number of GPUs cannot be greater than number of blocks.");
    if (p.run_l0_job || p.run_l1 || p.split_jobs) throw Fail("--gpus N shards one run; it cannot be combined with --split-l0 / --run-l0 / --run-l1.");
    log << " * sharding level 0 over " << G << " GPUs (blocks), level 1 by phenotype\n";
  }
  phase("inputs parsed");
  require_device();
  phase("cuda context");
  std::vector<rg_handle> hs(G, nullptr);
  struct HandlesGuard {
    std::vector<rg_handle>& v;
    ~HandlesGuard() { for (auto& x : v) { if (x && !g_fast_exit) rg_destroy(x); x = nullptr; } }
  } guards{hs};
  for (int d = 0; d < G; ++d) {
    cfg.device = (G > 1 ? d : p.gpu);
    rg_check(rg_step1_create(&cfg, ph.X.data(), ph.Y.data(), ph.mask.data(), ph.in_analysis.data(),
                             p.loocv ? nullptr : folds.data(), lambda.data(), ph.neff.data(), &hs[d]));
  }
  rg_handle h = hs[0];
  phase("rg_step1_create");
  std::vector<std::vector<uint8_t>> owned(G, std::vector<uint8_t>(P, 0));
  if (G > 1) {
    for (int i = 0; i < P; ++i) owned[i % G][i] = 1;
    for (int d = 0; d < G; ++d) rg_check(rg_W_set_owned(hs[d], owned[d].data()));
    for (int d = 0; d < G; ++d)
      for (int e = 0; e < G; ++e)
        if (e != d) rg_check(rg_W_attach_local(hs[d], hs[e], owned[e].data()));
  }
  auto owner_of = [&](int ph_i) { return hs[G > 1 ? ph_i % G : 0]; };

  // --l1-phenoList (with --run-l1): level 1 only for the named phenotypes (select_pheno_l1, src/Regenie.cpp:862-868)
  std::vector<uint8_t> l1_sel(P, 1);
  if (p.run_l1 && !p.l1_phenos.empty()) {
    bool any = false;
    for (int i = 0; i < P; ++i) { l1_sel[i] = p.l1_phenos.count(ph.names[i]) ? 1 : 0; any |= l1_sel[i] != 0; }
    if (!any) throw Fail("none of the phenotypes in --l1-phenoList is in the phenotype file.");
    rg_check(rg_l1_select(h, l1_sel.data()));
  }

  // ---- level 0
  std::vector<uint8_t> rows(use_bgen ? 0 : (size_t)p.bsize * g.row_stride);
  const bool subset = g.keys.size() != g.n_file;
  int last_chr = -1;
  const double t0 = now_ms();
  if (p.run_l1) {
    // read_l0 / read_l0_chunk (src/Step1_Models.cpp:1921-1987): columns [bstart*R, (bstart+btot)*R) from every job file
    log << " (skipping to level 1 models)\n";
    std::vector<double> slab((size_t)N * p.l0);
    for (int ph_i = 0; ph_i < P; ++ph_i) {
      if (!l1_sel[ph_i]) continue;
      int b0 = 0;
      for (const auto& mj : master.jobs) {
        const std::string fin = mj.prefix + "_l0_Y" + std::to_string(ph_i + 1);
        std::ifstream f(fin, std::ios::binary | std::ios::ate);
        if (!f) throw Fail("cannot open file : " + fin);
        if ((uint64_t)f.tellg() != (uint64_t)sizeof(double) * N * p.l0 * mj.nblocks) throw Fail("file " + fin + " is not the right size.");
        f.seekg(0);
        for (int b = 0; b < mj.nblocks; ++b) {
          f.read(reinterpret_cast<char*>(slab.data()), (std::streamsize)(slab.size() * sizeof(double)));
          rg_check(rg_l0_load_W(owner_of(ph_i), b0 + b, ph_i, slab.data()));
        }
        b0 += mj.nblocks;
      }
    }
  }
  // reader threads fetch blocks b+1 and b+2 from the file while block b is handed to the GPU (three buffers in rotation).
  // .bed rows sit in PINNED buffers (rg_host_alloc), so a block crosses PCIe by DMA straight from the buffer the reader
  // filled (a pageable buffer is first copied into the driver's staging area, ~5 ms per 25 MB block); rg_l0_wait_input
  // after each call tells when the buffer may be refilled.  Pageable inputs (.bgen bytes, .pgen records) are staged
  // before their call returns and can be refilled at once.
  constexpr int kBuf = 3, kAhead = 2;
  struct PinnedSet {
    void* p[kBuf] = {nullptr, nullptr, nullptr};
    ~PinnedSet() { for (void* q : p) if (q && !g_fast_exit) rg_host_free(q); }
  } pinned;
  std::vector<uint8_t> rows_extra[kBuf];
  uint8_t* bufs[kBuf] = {rows.data(), nullptr, nullptr};
  bool pin_rows = !use_bgen && !p.run_l1 && G == 1 && !rows.empty() && !(gbed.pg && pgen_on_device());
  for (int k = 0; k < kBuf && pin_rows; ++k) pin_rows = rg_host_alloc(&pinned.p[k], (int64_t)rows.size()) == 0;
  for (int k = 0; k < kBuf; ++k) {
    if (pin_rows) bufs[k] = (uint8_t*)pinned.p[k];
    else if (k > 0) { rows_extra[k].resize(rows.size()); bufs[k] = rows_extra[k].data(); }
  }
  std::vector<uint8_t> probs[kBuf], pmiss[kBuf];               // .bgen: inflated probability pairs + ploidy bytes of a block
  if (use_bgen && !p.run_l1)
    for (int k = 0; k < kBuf; ++k) { probs[k].resize((size_t)p.bsize * g.n_file * 2); pmiss[k].resize((size_t)p.bsize * g.n_file); }
  const int io_threads = std::max(1, std::min(32, (int)std::thread::hardware_concurrency()));
  const bool pgen_dev = !use_bgen && gbed.pg && pgen_on_device();
  if (pgen_dev) log << " * pgen records are decoded on the GPU\n";
  PgenBatch pbatch[kBuf];
  std::future<void> pending[kBuf];
  auto fetch = [&](int b) {
    return std::async(std::launch::async, [&, b] {
      const int k = b % kBuf;
      if (use_bgen) gg.read_block(blocks[b].first, blocks[b].size, probs[k].data(), pmiss[k].data(), io_threads);
      else if (pgen_dev) gbed.pg->gather(blocks[b].first, blocks[b].size, pbatch[k]);
      else gbed.read_rows(blocks[b].first, blocks[b].size, bufs[k]);
    });
  };
  if (G == 1) {
    // two reads in flight only where the reader is re-entrant (pread on the .bed, the in-memory .pgen); the .bgen reader
    // and the stream fallback of the .bed reader share a file cursor
    const int ahead = (use_bgen || (!gbed.pg && gbed.bed_fd < 0)) ? 1 : kAhead;
    for (int b = 0; b < ahead && b < nb && !p.run_l1; ++b) pending[b % kBuf] = fetch(b);
    for (int b = 0; b < nb && !p.run_l1; ++b) {
      if (blocks[b].chrom != last_chr) { log << "Chromosome " << blocks[b].chrom << "\n"; last_chr = blocks[b].chrom; }
      const int k = b % kBuf;
      pending[k].get();
      if (b + ahead < nb) pending[(b + ahead) % kBuf] = fetch(b + ahead);      // its buffer was block b-1's (or b's own slot + 1): consumed
      if (use_bgen)
        rg_check(rg_l0_block_dosage_u8(h, probs[k].data(), pmiss[k].data(), (int64_t)g.n_file, blocks[b].size,
                                       subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
      else if (pgen_dev) {
        const uint8_t* drows = nullptr;
        int64_t dstride = 0;
        pgen_rows_device(h, pbatch[k], blocks[b].size, (int64_t)gbed.pg->n_file, b, &drows, &dstride);
        rg_check(rg_l0_block_bed(h, drows, dstride, blocks[b].size, subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
      } else {
        rg_check(rg_l0_block_bed(h, bufs[k], (int64_t)g.row_stride, blocks[b].size,
                                 subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
        if (pin_rows) rg_check(rg_l0_wait_input(h));
      }
      log << " block [" << b + 1 << "] : " << blocks[b].size << " snps\n";
    }
  } else {
    // one host thread per GPU, each feeding its contiguous block range; the .bed stream is shared, so reads take a lock
    std::mutex io_mu, log_mu;
    std::vector<std::string> errs(G);
    std::vector<std::thread> workers;
    const int nall = nb / G, rem = nb - nall * G;
    int b0 = 0;
    for (int d = 0; d < G; ++d) {
      const int cnt = nall + (d < rem ? 1 : 0), first = b0;
      b0 += cnt;
      workers.emplace_back([&, d, first, cnt] {
        try {
          std::vector<uint8_t> buf(use_bgen ? 0 : (size_t)p.bsize * g.row_stride), pr, pm;
          if (use_bgen) { pr.resize((size_t)p.bsize * g.n_file * 2); pm.resize((size_t)p.bsize * g.n_file); }
          for (int b = first; b < first + cnt; ++b) {
            if (use_bgen) {
              gg.read_block(blocks[b].first, blocks[b].size, pr.data(), pm.data(), std::max(1, io_threads / G));
              rg_check(rg_l0_block_dosage_u8(hs[d], pr.data(), pm.data(), (int64_t)g.n_file, blocks[b].size,
                                             subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
            } else if (pgen_dev) {
              PgenBatch pb;                                  // gather only reads the mapped file: no lock
              gbed.pg->gather(blocks[b].first, blocks[b].size, pb);
              const uint8_t* drows = nullptr;
              int64_t dstride = 0;
              pgen_rows_device(hs[d], pb, blocks[b].size, (int64_t)gbed.pg->n_file, b, &drows, &dstride);
              rg_check(rg_l0_block_bed(hs[d], drows, dstride, blocks[b].size, subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
            } else {
              { std::lock_guard<std::mutex> lk(io_mu); gbed.read_rows(blocks[b].first, blocks[b].size, buf.data()); }
              rg_check(rg_l0_block_bed(hs[d], buf.data(), (int64_t)g.row_stride, blocks[b].size,
                                       subset ? g.sample_idx.data() : nullptr, p.ref_first, b));
            }
            std::lock_guard<std::mutex> lk(log_mu);
            log << " block [" << b + 1 << "] : " << blocks[b].size << " snps (gpu " << d << ")\n";
          }
        } catch (const Fail& f) { errs[d] = f.what(); }
        catch (const std::exception& e) { errs[d] = e.what(); }
      });
    }
    for (auto& w : workers) w.join();
    for (int d = 0; d < G; ++d) if (!errs[d].empty()) throw Fail(errs[d]);
  }
  for (int d = 0; d < G; ++d) {
    const int64_t st = rg_l0_status(hs[d]);
    if (st != 0) {
      if (st > 0 && st < (1ll << 40))
        throw Fail("!! Uh-oh, SNP " + g.snps[blocks[(st - 1) / p.bsize].first + (st - 1) % p.bsize].id + " has low variance.");
      throw Fail(std::string(rg_last_error()));
    }
  }
  log << " Level 0 done (" << (long)(now_ms() - t0) << "ms)\n";
  phase("level 0");
  if ((p.lowmem && p.keep_l0) || p.run_l0_job) {
    // write_l0_file (src/Step1_Models.cpp:728-733): per phenotype, per block an N x R column-major f64 slab.
    // The reference deletes these after level 1 unless --keep-l0 (src/Data.cpp:1011,1108,1131-1137); here W
    // never leaves HBM for level 1, so the files are only materialised when they are kept.
    const std::string pfx = p.lowmem_prefix.empty() ? p.out : p.lowmem_prefix;
    log << "   -files will have prefix [" << pfx << "_l0_Y]\n";
    std::vector<double> slab((size_t)N * p.l0);
    for (int ph_i = 0; ph_i < P; ++ph_i) {
      std::ofstream f(pfx + "_l0_Y" + std::to_string(ph_i + 1), std::ios::binary);
      if (!f) throw Fail("cannot write temporary file " + pfx + "_l0_Y" + std::to_string(ph_i + 1));
      for (int b = 0; b < nb; ++b) {
        rg_check(rg_l0_fetch_W(owner_of(ph_i), b, ph_i, slab.data()));
        f.write(reinterpret_cast<const char*>(slab.data()), (std::streamsize)(slab.size() * sizeof(double)));
      }
    }
  }
  if (p.run_l0_job) {
    log << "\nDone writing level 0 predictions to file.\n";
    return;
  }
  log << "\n Level 1 ridge...\n";

  // ---- level 1 (tau = B(1-h)/h, src/Step1_Models.cpp:2115)
  const double B = (double)nb * p.l0;
  std::vector<double> tau((size_t)P * p.l1), cs((size_t)5 * P * p.l1);
  const double tau_mult = p.bt ? 3.0 / (M_PI * M_PI) : 1.0;                     // src/Step1_Models.cpp:2115-2117
  for (int ph_i = 0; ph_i < P; ++ph_i)
    for (int j = 0; j < p.l1; ++j) tau[(size_t)ph_i * p.l1 + j] = B * (1 - h1[j]) / h1[j] * tau_mult;
  std::vector<int32_t> best(P);
  std::vector<double> bt_offs;
  if (p.bt) {
    // offset_nullreg: covariate-only logistic fit per trait (fit_null_logistic, src/Step1_Models.cpp:54-140)
    std::vector<double> offs((size_t)N * P);
    for (int ph_i = 0; ph_i < P; ++ph_i) {
      const std::vector<double> eta = null_logistic_eta(ph.names[ph_i], &ph.Y_raw[(size_t)ph_i * N], ph.X.data(), N, ph.C,
                                                        &ph.mask[(size_t)ph_i * N]);
      std::copy(eta.begin(), eta.end(), offs.begin() + (size_t)ph_i * N);
    }
    cs.assign((size_t)6 * P * p.l1, 0.0);
    if (G == 1) rg_check(rg_l1_fit_bt(h, ph.Y_raw.data(), offs.data(), tau.data(), cs.data(), best.data()));
    else bt_offs = offs;
  } else if (G == 1) {
    rg_check(rg_l1_fit(h, tau.data(), cs.data(), best.data()));
  }
  phase("level 1");
  std::vector<int32_t> chr_of_block(nb);
  for (int b = 0; b < nb; ++b) chr_of_block[b] = blocks[b].chrom;
  std::vector<double> loco((size_t)P * 23 * N);
  if (G == 1) {
    rg_check(rg_loco(h, chr_of_block.data(), loco.data()));
  } else {
    // every GPU fits and assembles the phenotypes it owns, concurrently; the host merges disjoint supports
    std::vector<std::string> errs(G);
    std::vector<std::vector<double>> cs_d(G, std::vector<double>(cs.size(), 0.0)), loco_d(G);
    std::vector<std::vector<int32_t>> best_d(G, std::vector<int32_t>(P, 0));
    std::vector<std::thread> workers;
    for (int d = 0; d < G; ++d)
      workers.emplace_back([&, d] {
        try {
          if (p.bt) rg_check(rg_l1_fit_bt(hs[d], ph.Y_raw.data(), bt_offs.data(), tau.data(), cs_d[d].data(), best_d[d].data()));
          else rg_check(rg_l1_fit(hs[d], tau.data(), cs_d[d].data(), best_d[d].data()));
          loco_d[d].assign((size_t)P * 23 * N, 0.0);
          rg_check(rg_loco(hs[d], chr_of_block.data(), loco_d[d].data()));
        } catch (const Fail& f) { errs[d] = f.what(); }
        catch (const std::exception& e) { errs[d] = e.what(); }
      });
    for (auto& w : workers) w.join();
    for (int d = 0; d < G; ++d) if (!errs[d].empty()) throw Fail(errs[d]);
    const int nsum = (int)(cs.size() / ((size_t)P * p.l1));
    for (int ph_i = 0; ph_i < P; ++ph_i) {
      const int d = ph_i % G;
      best[ph_i] = best_d[d][ph_i];
      for (int k = 0; k < nsum; ++k)
        for (int j = 0; j < p.l1; ++j) cs[((size_t)k * P + ph_i) * p.l1 + j] = cs_d[d][((size_t)k * P + ph_i) * p.l1 + j];
      std::copy(loco_d[d].begin() + (size_t)ph_i * 23 * N, loco_d[d].begin() + (size_t)(ph_i + 1) * 23 * N,
                loco.begin() + (size_t)ph_i * 23 * N);
    }
  }

  // ---- output (Data::output src/Data.cpp:956-1120, write_predictions :1795-1982)
  log << "Output\n------\n";
  std::ofstream plist(p.out + "_pred.list"), prs_list;
  if (!plist) throw Fail("cannot write to file : " + p.out + "_pred.list");
  std::vector<double> prs;
  if (p.print_prs) {                                         // whole-genome PRS next to the LOCO files (src/Data.cpp:1906-1922)
    prs_list.open(p.out + "_prs.list");
    if (!prs_list) throw Fail("cannot write to file : " + p.out + "_prs.list");
    prs.resize((size_t)P * N);
    if (G == 1) {
      rg_check(rg_prs(h, prs.data()));
    } else {
      std::vector<double> tmp((size_t)P * N);
      for (int d = 0; d < G; ++d) {
        rg_check(rg_prs(hs[d], tmp.data()));
        for (int ph_i = d; ph_i < P; ph_i += G) std::copy(tmp.begin() + (size_t)ph_i * N, tmp.begin() + (size_t)(ph_i + 1) * N, prs.begin() + (size_t)ph_i * N);
      }
    }
  }
  const std::string gz_ext = p.gz ? ".gz" : "";
  std::vector<uint32_t> order;             // std::map key order of FID_IID, analysed samples only
  for (auto& kv : g.key_to_ind) if (ph.in_analysis[kv.second]) order.push_back(kv.second);
  std::vector<int> chr_labels(23);
  for (int c = 0; c < 23; ++c) chr_labels[c] = c + 1;
  phase("loco assembled");
  for (int ph_i = 0; ph_i < P; ++ph_i) {
    if (!l1_sel[ph_i]) continue;
    log << "phenotype " << ph_i + 1 << " (" << ph.names[ph_i] << ") : \n";
    auto CS = [&](int k, int j) { return cs[((size_t)k * P + ph_i) * p.l1 + j]; };
    const double ne = ph.neff[ph_i];
    for (int j = 0; j < p.l1; ++j) {
      double num = CS(4, j) - CS(0, j) * CS(1, j) / ne;
      const double rsq = num * num / ((CS(2, j) - CS(0, j) * CS(0, j) / ne) * (CS(3, j) - CS(1, j) * CS(1, j) / ne));
      const double sse = CS(2, j) + CS(3, j) - 2 * CS(4, j);
      std::ostringstream l;
      const double tj = tau[(size_t)ph_i * p.l1 + j];
      l << "  " << std::setw(5) << (p.bt ? B / (B + (M_PI * M_PI / 3.0) * tj) : B / (B + tj)) << " : Rsq = " << rsq
        << ", MSE = " << sse / ne;
      if (p.bt) l << ", -logLik/N = " << CS(5, j) / ne;
      l << (j == best[ph_i] ? "<- min value" : "");
      log << l.str() << "\n";
    }
    const uint8_t* mask_p = &ph.mask[(size_t)ph_i * N];
    const std::string loco_file = p.out + "_" + std::to_string(ph_i + 1) + ".loco" + gz_ext;
    {
      TextWriter of;
      of.open(loco_file);
      const double* L = loco.data() + (size_t)ph_i * 23 * N;
      std::vector<const double*> chr_rows(23);
      for (int c = 0; c < 23; ++c) chr_rows[c] = L + (size_t)c * N;
      write_pred_file(of, g.keys, order, mask_p, chr_labels, chr_rows);
      of.close();
    }
    plist << ph.names[ph_i] << " " << full_path(loco_file, p.rel_path) << "\n";
    log << "  * making predictions...writing LOCO predictions...";
    if (p.print_prs) {
      const std::string prs_file = p.out + "_" + std::to_string(ph_i + 1) + ".prs" + gz_ext;
      TextWriter of;
      of.open(prs_file);
      write_pred_file(of, g.keys, order, mask_p, {0}, {prs.data() + (size_t)ph_i * N});
      of.close();
      prs_list << ph.names[ph_i] << " " << full_path(prs_file, p.rel_path) << "\n";
      log << "writing whole genome PRS...";
    }
    log << "done\n\n";
  }
  if (p.write_null_firth && p.bt) {
    // null approximate-Firth estimates per chromosome, warm-started along the chromosomes (src/Data.cpp:1873-1903); they are
    // starting values for Step 2 (--use-null-firth), not results
    std::ofstream flist(p.out + "_firth.list");
    if (!flist) throw Fail("cannot write to file : " + p.out + "_firth.list");
    for (int ph_i = 0; ph_i < P; ++ph_i) {
      if (!l1_sel[ph_i]) continue;
      const std::string ffile = p.out + "_" + std::to_string(ph_i + 1) + ".firth" + gz_ext;
      std::vector<double> bhat = null_logistic_beta(ph.names[ph_i], &ph.Y_raw[(size_t)ph_i * N], ph.X.data(), N, ph.C,
                                                    &ph.mask[(size_t)ph_i * N]);
      std::string text;
      bool ok = true;
      char num[40];
      for (int c = 0; c < 23 && ok; ++c) {
        ok = fit_null_firth(&ph.Y_raw[(size_t)ph_i * N], ph.X.data(), N, ph.C, loco.data() + ((size_t)ph_i * 23 + c) * N,
                            &ph.mask[(size_t)ph_i * N], bhat);
        text += std::to_string(c + 1);
        for (double v : bhat) text.append(num, (size_t)snprintf(num, sizeof(num), " %g", v));
        text += '\n';
      }
      if (!ok) { log << "WARNING: Firth failed to converge for phenotype '" << ph.names[ph_i] << "'\n"; continue; }
      TextWriter of;
      of.open(ffile);
      of << text;
      of.close();
      flist << ph.names[ph_i] << " " << full_path(ffile, p.rel_path) << "\n";
    }
    flist.close();
    log << "List of files with null Firth estimates written to: [" << p.out << "_firth.list]\n";
  }
  plist.close();
  phase("prediction files");
  if (p.run_l1 && !p.keep_l0)                        // rm_l0_files (src/Data.cpp:1131-1147)
    for (const auto& mj : master.jobs) {
      for (int ph_i = 0; ph_i < P; ++ph_i) remove((mj.prefix + "_l0_Y" + std::to_string(ph_i + 1)).c_str());
      remove((mj.prefix + ".snplist").c_str());
    }
  log << "List of blup files written to: [" << p.out << "_pred.list]\n";
  if (p.print_prs) {
    prs_list.close();
    log << "List of files with whole genome PRS written to: [" << p.out << "_prs.list]\n";
  }
}

// ------------------------------------------------------------------------------------ step 2
// --test dominant | recessive (parseSnpfromBed src/Geno.cpp:2509-2530, BGEN :2084-2125): allele frequency, INFO, N and the
// MAC filters come from the additive coding; the genotypes are then recoded (dominant: 2 -> 1, recessive: 1 -> 0 and
// 2 -> 1; on dosages P(het) + P(hom) and P(hom)) and the test runs on the recoded values, with no minor-allele flip
// (src/Data.cpp:2108).  Here: a first pass over the block yields the additive counts, the input bytes are recoded on the
// host so that the unchanged kernels see the recoded genotype, and a second pass (no MAC filter) yields the test.
struct Recode {
  uint8_t lut[256];
  int type = 0;
  bool ref_first = false;
  Recode(int type_, bool ref_first_) : type(type_), ref_first(ref_first_) {
    // PLINK 1 codes: 00 = two copies of the first .bim allele, 10 = one, 11 = none, 01 = missing.  The kernels count
    // the first allele (ref-last) or 2 minus that (--ref-first), so "two copies of the effect allele" is 00 or 11.
    int map[4] = {0, 1, 2, 3};
    const int two = ref_first ? 3 : 0, none = ref_first ? 0 : 3;
    if (type == 1) map[two] = 2;                       // dominant: 2 -> 1
    if (type == 2) { map[two] = 2; map[2] = none; }    // recessive: 2 -> 1, 1 -> 0
    for (int b = 0; b < 256; ++b) {
      int o = 0;
      for (int k = 0; k < 4; ++k) o |= map[(b >> (2 * k)) & 3] << (2 * k);
      lut[b] = (uint8_t)o;
    }
  }
  void bed(uint8_t* rows, size_t nbytes) const {
    for (size_t i = 0; i < nbytes; ++i) rows[i] = lut[rows[i]];
  }
  // 8-bit probability pairs (p0, p1) of the first-allele homozygote and the heterozygote; the kernels form
  // p1 + 2 p0 (ref-last) or p1 + 2 (255 - p0 - p1) (--ref-first).  The recoded value t goes into p1, with p0 chosen so
  // that the homozygote term vanishes.
  void probs(uint8_t* pr, size_t n_pairs) const {
    for (size_t i = 0; i < n_pairs; ++i) {
      const int p0 = pr[2 * i], p1 = pr[2 * i + 1], p2 = std::max(0, 255 - p0 - p1);
      const int hom = ref_first ? p2 : p0;
      const int t = type == 1 ? std::min(255, hom + p1) : hom;
      pr[2 * i + 1] = (uint8_t)t;
      pr[2 * i] = ref_first ? (uint8_t)(255 - t) : 0;
    }
  }
};

const char* test_name(int test_type) { return test_type == 1 ? "DOM" : test_type == 2 ? "REC" : "ADD"; }

// flags of the two passes: bit 0 (MAC) from the additive pass, everything else from the pass on the recoded genotypes,
// plus `total < numtol` on the recoded mean (src/Geno.cpp:2523-2527)
void merge_recode_flags(int bs, int32_t* flags, const int32_t* flags2, const double* af_all2) {
  for (int v = 0; v < bs; ++v) {
    flags[v] = (flags[v] & 1) | (flags2[v] & ~1);
    if (2.0 * af_all2[v] < 1e-6) flags[v] |= 1;
  }
}

// Step-2 output files: one per trait (setup_output, split mode, src/Data.cpp:2026-2035) or, with --no-split, one file
// for all traits plus the <out>.regenie.Ydict dictionary (src/Data.cpp:2011-2022).  Rows are collected per block.
struct S2Writers {
  bool no_split = false;
  std::vector<TextWriter> outs;
  TextWriter all;
  std::vector<std::string> obuf;
  std::string obuf_all;
  void open(const Params& p, const Pheno& ph, bool with_info) {
    no_split = p.no_split;
    const std::string gz_ext = p.gz ? ".gz" : "";
    obuf.resize(ph.P);
    if (no_split) {
      all.open(p.out + ".regenie" + gz_ext);
      all << sumstats_header_all(ph.P, with_info);
      TextWriter dict;
      dict.open(p.out + ".regenie.Ydict");
      for (int i = 0; i < ph.P; ++i) dict << ("Y" + std::to_string(i + 1) + " " + ph.names[i] + "\n");
      dict.close();
      return;
    }
    outs = std::vector<TextWriter>(ph.P);
    for (int i = 0; i < ph.P; ++i) {
      outs[i].open(p.out + "_" + ph.names[i] + ".regenie" + gz_ext);
      outs[i] << (p.htp ? htp_header() : sumstats_header(with_info, p.af_cc));
    }
  }
  void flush() {
    if (no_split) { all << obuf_all; obuf_all.clear(); return; }
    for (size_t i = 0; i < outs.size(); ++i) { outs[i] << obuf[i]; obuf[i].clear(); }
  }
  void close() {
    flush();
    if (no_split) all.close();
    for (auto& o : outs) o.close();
  }
};

// --no-split prints N_RR N_RA N_AA of all analysed samples (src/Geno.cpp:2480-2486).  For hard calls they follow from two
// allele sums the kernels already return: a pass over the block recoded as "recessive" (1 -> 0, 2 -> 1) counts the
// homozygotes, N_AA = sum of the recoded genotypes; with S = 2 N A1FREQ the additive sum, N_RA = S - 2 N_AA and
// N_RR = N - N_RA - N_AA.  The pass runs before the test passes so that the block left on the device is the tested one.
struct GenoCounts {
  bool on = false;
  Recode rec;
  std::vector<uint8_t> rows;
  std::vector<double> af, mac, af_all, mac_all, stat, beta, se, chisq, scale;
  std::vector<int32_t> ns, ns_all, flags;
  std::vector<long> n_aa;
  rg_s2_out out;
  GenoCounts(bool on_, int bsz, int P, size_t row_bytes, bool ref_first) : on(on_), rec(2, ref_first) {
    if (on) {
      rows.resize((size_t)bsz * row_bytes);
      const size_t bp = (size_t)bsz * P;
      af.resize(bp); mac.resize(bp); stat.resize(bp); beta.resize(bp); se.resize(bp); chisq.resize(bp); ns.resize(bp);
      af_all.resize(bsz); mac_all.resize(bsz); scale.resize(bsz); ns_all.resize(bsz); flags.resize(bsz); n_aa.resize(bsz);
    }
    out = rg_s2_out{af.data(), ns.data(), mac.data(), af_all.data(), ns_all.data(), mac_all.data(), flags.data(),
                    scale.data(), stat.data(), beta.data(), se.data(), chisq.data()};
  }
  // `call(rows, &out)` runs the block entry point on the recoded copy with the MAC filter off
  template <typename Call>
  void run(const uint8_t* src, size_t nbytes, int bs, Call&& call) {
    if (!on) return;
    memcpy(rows.data(), src, nbytes);
    rec.bed(rows.data(), nbytes);
    call(rows.data(), &out);
    for (int v = 0; v < bs; ++v) n_aa[v] = std::lround(2.0 * af_all[v] * ns_all[v]);
  }
  // N_RR, N_RA, N_AA of variant v given the additive pass
  void counts(int v, double af_add, int n, long& n_rr, long& n_ra, long& n_aa_out) const {
    const long s = std::lround(2.0 * af_add * n);
    n_aa_out = n_aa[v];
    n_ra = s - 2 * n_aa_out;
    n_rr = n - n_ra - n_aa_out;
  }
};

// --htp on hard calls: the genotype counts of each trait's samples (update_genocounts, src/Geno.cpp:2986-3018: rows 0-2 =
// cases - all samples of a quantitative trait -, rows 3-5 = controls) straight from the 2-bit rows on the host: per
// (trait, class) a sample mask in FILE order with one bit per 2-bit field, three popcounts per 32 samples.  On the
// non-PAR part of chromosome X the reference counts a male with g >= 1 as alt and any other male call as ref; females and
// everything else: het / alt as they are, missing calls skipped.
struct BedTraitCounts {
  int P = 0;
  bool binary = false, ref_first = false;
  size_t words = 0;
  std::vector<uint64_t> m_all, m_male;                       // [P][2 classes][words]
  size_t at(int p, int c) const { return ((size_t)p * 2 + c) * words; }
  // cls [P][N] in kept-sample order: 0 = not in the trait, 1 = in the trait (control of a binary trait), 2 = case
  void init(int P_, bool binary_, bool ref_first_, size_t n_file, const std::vector<int32_t>& sample_idx, const uint8_t* cls,
            const uint8_t* male) {
    P = P_; binary = binary_; ref_first = ref_first_;
    words = (n_file + 31) / 32;
    m_all.assign((size_t)P * 2 * words, 0);
    m_male.assign((size_t)P * 2 * words, 0);
    const size_t N = sample_idx.size();
    for (int p = 0; p < P; ++p)
      for (size_t k = 0; k < N; ++k) {
        const int c = cls[(size_t)p * N + k];
        if (!c) continue;
        const size_t f = (size_t)sample_idx[k];
        const uint64_t bit = 1ull << (2 * (f % 32));
        m_all[at(p, c - 1) + f / 32] |= bit;
        if (male && male[k]) m_male[at(p, c - 1) + f / 32] |= bit;
      }
  }
  // out [bs][P][6]; non_par [bs] or null
  void count(const uint8_t* rows, size_t row_stride, int bs, const uint8_t* non_par, long* out, int threads) const {
    std::atomic<int> next{0};
    auto work = [&]() {
      std::vector<long> c((size_t)P * 2 * 6);                // [trait][class][all: het, two, none | male: het, two, none]
      for (;;) {
        const int v = next.fetch_add(1);
        if (v >= bs) return;
        const uint8_t* r = rows + (size_t)v * row_stride;
        const bool np = non_par && non_par[v];
        std::fill(c.begin(), c.end(), 0);
        for (size_t w = 0; w < words; ++w) {
          uint64_t x = 0;
          const size_t off = w * 8, nb = off + 8 <= row_stride ? 8 : row_stride - off;
          memcpy(&x, r + off, nb);                           // little endian: field s of the word = sample 32 w + s
          const uint64_t lo = x & 0x5555555555555555ull, hi = (x >> 1) & 0x5555555555555555ull;
          const uint64_t het = hi & ~lo, c11 = hi & lo, c00 = ~hi & ~lo & 0x5555555555555555ull;   // 01 = missing
          for (int pc = 0; pc < 2 * P; ++pc) {
            const uint64_t ma = m_all[(size_t)pc * words + w];
            if (!ma) continue;
            long* cc = &c[(size_t)pc * 6];
            cc[0] += __builtin_popcountll(het & ma); cc[1] += __builtin_popcountll(c00 & ma); cc[2] += __builtin_popcountll(c11 & ma);
            if (np) {
              const uint64_t mm = m_male[(size_t)pc * words + w];
              cc[3] += __builtin_popcountll(het & mm); cc[4] += __builtin_popcountll(c00 & mm); cc[5] += __builtin_popcountll(c11 & mm);
            }
          }
        }
        long* o = out + (size_t)v * P * 6;
        for (int p = 0; p < P; ++p)
          for (int k = 0; k < 2; ++k) {                       // k = 0: the "cases" columns, 1: the "controls" columns
            long* t = o + p * 6 + 3 * k;
            if (k == 1 && !binary) { t[0] = t[1] = t[2] = 0; continue; }
            const long* cc = &c[((size_t)p * 2 + (binary ? 1 - k : 0)) * 6];   // class 2 (cases) first for a binary trait
            // code 00 = two copies of the first .bim allele: the counted allele unless --ref-first (see Recode)
            const long het = cc[0], alt = ref_first ? cc[2] : cc[1], ref = ref_first ? cc[1] : cc[2];
            const long het_m = cc[3];
            t[0] = ref; t[1] = het - het_m; t[2] = alt + het_m;  // non-PAR males: g >= 1 -> alt (het_m = 0 elsewhere)
          }
      }
    };
    const int T = std::max(1, std::min(threads, bs));
    std::vector<std::thread> pool;
    for (int t = 1; t < T; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
  }
};

// --range (in_range, src/Geno.cpp:2790-2800): keep the variants of one chromosome window
void apply_range(const Params& p, std::vector<Snp>& snps) {
  if (!p.set_range) return;
  snps.erase(std::remove_if(snps.begin(), snps.end(), [&](const Snp& s) {
               return s.chrom != p.range_chr || (double)s.pos < p.range_min || (double)s.pos > p.range_max;
             }), snps.end());
}

// phenotypes + covariates + LOCO files for Step 2 (read_pheno_and_cov, blup_read, prep_run)
void load_step2_inputs(const Params& p, const SampleSet& g, const std::vector<std::pair<std::string, std::string>>& ids_file,
                       const std::vector<int32_t>& sample_idx, Pheno& ph, std::vector<Loco>& locos, Log& log) {
  ph.pheno_cols = p.pheno_cols; ph.covar_cols = p.covar_cols; ph.rint = p.rint && !p.bt; ph.cat_cols = p.cat_cols; ph.max_cat_levels = p.max_cat_levels;
  ph.pheno_excl = p.pheno_excl; ph.covar_excl = p.covar_excl; ph.min_case_count = p.min_case_count;
  read_pheno_and_cov(g, p.pheno, p.covar, true, p.strict, p.bt, ph, log);
  const int64_t N = ph.N;
  const int P = ph.P;
  // write_ids (src/Pheno.cpp:1538-1576) runs right after blup_read, before setMasks: the samples with a phenotype
  // value and a prediction
  auto write_ids = [&](const std::vector<uint8_t>* extra) {
    if (!p.write_samples) return;
    log << " * user specified to write sample IDs for each trait\n";
    std::vector<std::pair<std::string, std::string>> kept(N);
    for (int64_t s = 0; s < N; ++s) kept[s] = ids_file.at((size_t)sample_idx[s]);
    std::vector<uint8_t> m(N);
    for (int i = 0; i < P; ++i) {
      for (int64_t s = 0; s < N; ++s) m[s] = ph.mask[(size_t)i * N + s] && (!extra || (*extra)[(size_t)i * N + s]);
      write_ids_file(p.out + "_" + ph.names[i] + ".regenie.ids", ph.names[i], p.print_pheno, kept, m.data());
    }
  };
  if (p.ignore_pred) {                                      // --ignore-pred: no LOCO files, blup = 0 (src/Pheno.cpp:1060-1068)
    log << " * no step 1 predictions given. Simple " << (p.bt ? "logistic" : "linear") << " regression will be performed\n";
    locos.assign(P, Loco());
    write_ids(nullptr);
    prep_run(ph, nullptr, log);
    return;
  }
  log << " * " << (p.use_prs ? "PRS" : "LOCO") << " predictions : [" << p.pred << "]\n";
  const auto blup_files = read_pred_list(p.pred);
  locos.resize(P);
  std::vector<uint8_t> extra((size_t)N * P, 0);
  for (int i = 0; i < P; ++i) {
    auto it = blup_files.find(ph.names[i]);
    if (it == blup_files.end()) throw Fail("No step 1 file provided for phenotype '" + ph.names[i] + "'.");
    locos[i] = read_loco(it->second, p.use_prs);
    log << "   -file [" << it->second << "] for phenotype '" << ph.names[i] << "'\n";
    const auto& first = locos[i].first;                      // blup_read checks the first data row
    for (size_t c = 0; c < locos[i].ids.size(); ++c) {
      auto k = g.key_to_ind.find(locos[i].ids[c]);
      if (k == g.key_to_ind.end() || first.empty()) continue;
      extra[(size_t)i * N + k->second] = !std::isnan(first[c]);
    }
  }
  write_ids(&extra);
  prep_run(ph, &extra, log);
}

// blup_read_chr (src/Step2_Models.cpp:96-124): LOCO prediction of trait i for one chromosome
std::vector<double> blup_for_chr(Loco& loco, const SampleSet& g, const Pheno& ph, int i, int chrom) {
  const int64_t N = ph.N;
  std::vector<double> blup(N, 0.0);
  if (loco.empty()) return blup;                            // --ignore-pred
  if (!loco.has_row(chrom)) throw Fail("blup file for phenotype '" + ph.names[i] + "' has no row for chromosome " + std::to_string(chrom));
  const std::vector<double>& row = loco.row(chrom);          // --use-prs: the same whole-genome row for every chromosome
  for (size_t c = 0; c < loco.ids.size(); ++c) {
    auto k = g.key_to_ind.find(loco.ids[c]);
    if (k == g.key_to_ind.end()) continue;
    const uint32_t s = k->second;
    if (!ph.in_analysis[s] || !ph.mask[(size_t)i * N + s]) continue;
    if (std::isnan(row[c])) throw Fail("individual has missing predictions (FID_IID=" + loco.ids[c] + ")");
    blup[s] = row[c];
  }
  return blup;
}

// in_non_par (src/Geno.cpp:2802-2814) for the variants of one block; returns false when none is flagged
bool non_par_flags(const Params& p, const std::vector<Snp>& snps, const Block& b, std::vector<uint8_t>& flags) {
  flags.assign(b.size, 0);
  if (b.chrom != 23) return false;
  bool any = false;
  for (int v = 0; v < b.size; ++v) {
    const uint64_t pos = snps[b.first + v].pos;
    flags[v] = !(pos <= p.par1_max || pos >= p.par2_min);
    any |= flags[v] != 0;
  }
  return any;
}

// params.sex == 1 for the kept samples (read_fam / read_bgen_sample)
std::vector<uint8_t> male_vector(const std::vector<int>& sex_file, const std::vector<int32_t>& sample_idx) {
  std::vector<uint8_t> m(sample_idx.size(), 0);
  for (size_t i = 0; i < sample_idx.size(); ++i) m[i] = sex_file[sample_idx[i]] == 1;
  return m;
}

void run_step2_qt(const Params& p, Log& log) {
  const bool use_bgen = !p.bgen.empty();
  BedFile g;
  BgenFile gg;
  const auto excl = read_id_list(p.exclude, 1), extr = read_id_list(p.extract, 1), rem = read_id_list(p.remove, 2),
             keepl = read_id_list(p.keep, 2);
  if (use_bgen) {
    gg.sex_specific = p.sex_specific;
    gg.open(p.bgen, p.sample, p.ref_first, excl, extr, rem, keepl, p.chrs, p.bgi);
    if (gg.used_bgi) log << "   -index bgi file [" << (p.bgi.empty() ? p.bgen + ".bgi" : p.bgi) << "]\n";
    log << " * bgen                : [" << p.bgen << "] n_snps = " << gg.snps.size() << ", n_samples = " << gg.keys.size() << "\n";
  } else {
    open_rows(p, g, excl, extr, rem, keepl, log);
  }
  apply_range(p, gg.snps);
  apply_range(p, g.snps);
  if (g.pg) apply_range(p, g.pg->snps);
  if (p.set_range && (use_bgen ? gg.snps : g.snps).empty()) throw Fail("no variant left to include in analysis.");
  const std::vector<Snp>& snps = use_bgen ? gg.snps : g.snps;
  const std::vector<std::string>& keys = use_bgen ? gg.keys : g.keys;
  const std::vector<int32_t>& sample_idx = use_bgen ? gg.sample_idx : g.sample_idx;
  const size_t n_file = use_bgen ? gg.n_file : g.keys_file.size();
  const SampleSet ss{keys, use_bgen ? gg.key_to_ind : g.key_to_ind};
  Pheno ph;
  std::vector<Loco> locos;
  load_step2_inputs(p, ss, use_bgen ? gg.ids_file : g.ids_file, sample_idx, ph, locos, log);
  const int64_t N = ph.N;
  const int P = ph.P;
  const auto blocks = set_blocks(snps, p.bsize);
  log << " * # blocks            : [" << blocks.size() << "]\n";

  rg_step2_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.device = p.gpu; cfg.n_samples = N; cfg.n_cov = ph.C; cfg.n_pheno = P; cfg.max_block_size = p.bsize;
  cfg.n_analyzed = ph.n_analyzed; cfg.strict_mode = ph.strict;
  rg_handle h = nullptr;
  HandleGuard guard{h};
  require_device();
  rg_check(rg_step2_create(&cfg, ph.X.data(), ph.mask.data(), ph.in_analysis.data(), &h));

  S2Writers w;
  w.open(p, ph, use_bgen);
  std::vector<std::string>& obuf = w.obuf;                   // rows of the current block, one buffer per trait
  std::string head_s;
  const int bsz = p.bsize;
  GenoCounts gc(p.no_split, bsz, P, use_bgen ? 0 : g.row_stride, p.ref_first);
  // input blocks are fetched (file read / threaded BGEN inflate) one block ahead of the GPU call: the rg_s2_block_*
  // calls return with the results on the host, so the buffer of block b is free again when block b+2 is fetched
  std::vector<uint8_t> rows[2], probs[2], pmiss[2];
  for (int k = 0; k < 2; ++k) {
    if (use_bgen) { probs[k].resize((size_t)bsz * n_file * 2); pmiss[k].resize((size_t)bsz * n_file); }
    else rows[k].resize((size_t)bsz * g.row_stride);
  }
  const int threads = p.threads > 0 ? p.threads : (int)std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
  // --minINFO also drops a variant whose INFO over all analysed samples is too low (src/Geno.cpp:2074): computed from the
  // inflated bytes on the host, in the fetch thread
  const bool use_info1 = use_bgen && (p.min_info > 0 || p.no_split);   // --no-split prints it and the dosage genotype counts
  // --htp on dosages: thresholded genotype counts per trait (update_genocounts, src/Geno.cpp:2986-3018) from the inflated
  // bytes, in the fetch thread (BgenFile::trait_counts)
  // hard calls: the same counts by popcounts over the 2-bit rows (BedTraitCounts).  Both run in the fetch thread.
  const bool htp_bgen = use_bgen && p.htp;
  std::vector<uint8_t> htp_cls, htp_npf[2];
  const std::vector<uint8_t> htp_male = p.htp ? male_vector(use_bgen ? gg.sex_file : g.sex_file, sample_idx) : std::vector<uint8_t>();
  std::vector<long> htp_cnt[2];
  BedTraitCounts btc;
  if (p.htp) {
    htp_cls.resize((size_t)P * N);
    for (size_t e = 0; e < htp_cls.size(); ++e) htp_cls[e] = ph.mask[e] ? 1 : 0;
    for (int k = 0; k < 2; ++k) htp_cnt[k].resize((size_t)bsz * P * 6);
    if (!use_bgen) btc.init(P, false, p.ref_first, n_file, sample_idx, htp_cls.data(), htp_male.data());
  }
  const bool dev_inflate = use_bgen && p.gpu_inflate && gg.compression == 1 && p.test_type == 0 && !use_info1 && !htp_bgen;
  if (use_bgen && p.gpu_inflate)
    log << (dev_inflate ? " * bgen genotype blocks are inflated on the GPU\n"
                        : "   -WARNING: --gpu-inflate needs zlib-compressed payloads, the additive test and no --minINFO / --no-split / --htp; inflating on the host.\n");
  std::vector<uint8_t> comp[2];
  std::vector<uint64_t> comp_offs[2];
  std::vector<double> info1[2];
  std::vector<long> d_rr[2], d_aa[2];
  if (use_info1) for (int k = 0; k < 2; ++k) { info1[k].resize(bsz); d_rr[k].resize(bsz); d_aa[k].resize(bsz); }
  // .pgen records are expanded on the GPU unless an option edits the rows on the host (see pgen_on_device)
  const bool pgen_dev = !use_bgen && g.pg && pgen_on_device() && !p.no_split && !p.htp && p.test_type == 0;
  if (pgen_dev) log << " * pgen records are decoded on the GPU\n";
  PgenBatch pbatch[2];
  std::future<void> pending;
  auto fetch = [&](size_t b) {
    return std::async(std::launch::async, [&, b] {
      if (dev_inflate) gg.read_block_compressed(blocks[b].first, blocks[b].size, comp[b & 1], comp_offs[b & 1]);
      else if (use_bgen) {
        gg.read_block(blocks[b].first, blocks[b].size, probs[b & 1].data(), pmiss[b & 1].data(), threads);
        if (use_info1) gg.info_all(probs[b & 1].data(), pmiss[b & 1].data(), blocks[b].size, ph.in_analysis.data(), p.ref_first,
                                   info1[b & 1].data(), threads, d_rr[b & 1].data(), d_aa[b & 1].data());
        if (htp_bgen) {
          const bool np = non_par_flags(p, snps, blocks[b], htp_npf[b & 1]);
          gg.trait_counts(probs[b & 1].data(), pmiss[b & 1].data(), blocks[b].size, htp_cls.data(), P, false, p.ref_first,
                          htp_cnt[b & 1].data(), threads, htp_male.data(), np ? htp_npf[b & 1].data() : nullptr);
        }
      }
      else if (pgen_dev) g.pg->gather(blocks[b].first, blocks[b].size, pbatch[b & 1]);
      else {
        g.read_rows(blocks[b].first, blocks[b].size, rows[b & 1].data());
        if (p.htp) {
          const bool np = non_par_flags(p, snps, blocks[b], htp_npf[b & 1]);
          btc.count(rows[b & 1].data(), g.row_stride, blocks[b].size, np ? htp_npf[b & 1].data() : nullptr, htp_cnt[b & 1].data(), threads);
        }
      }
    });
  };
  if (blocks.empty()) throw Fail("no variant left to include in analysis.");
  if (p.start_block > (int)blocks.size()) throw Fail("Starting block > number of blocks analyzed");   // src/Data.cpp:2863-2864
  const size_t b_first = p.start_block > 1 ? (size_t)p.start_block - 1 : 0;
  if (b_first) log << "    + skipping to block #" << p.start_block << "\n";
  if (!blocks.empty()) pending = fetch(b_first);
  std::vector<double> info((size_t)bsz * P);
  std::vector<double> af((size_t)bsz * P), mac((size_t)bsz * P), stat((size_t)bsz * P), beta((size_t)bsz * P),
      se((size_t)bsz * P), chisq((size_t)bsz * P), af_all(bsz), mac_all(bsz), scale_fac(bsz);
  std::vector<int32_t> ns((size_t)bsz * P), ns_all(bsz), flags(bsz);
  rg_s2_out out{af.data(), ns.data(), mac.data(), af_all.data(), ns_all.data(), mac_all.data(), flags.data(),
                scale_fac.data(), stat.data(), beta.data(), se.data(), chisq.data()};
  const bool subset = keys.size() != n_file;
  // --htp: test_string + wgr_string + correction_type (src/Data.cpp:2075-2102)
  const std::string htp_model = std::string(test_name(p.test_type)) + (p.ignore_pred ? "" : "-WGR") + "-LR";
  // second pass of --test dominant / recessive: counts go to scratch, the test columns to the arrays that are printed
  const Recode recode(p.test_type, p.ref_first);
  std::vector<double> af2, mac2, af_all2, mac_all2, info2;
  std::vector<int32_t> ns2, ns_all2, flags2;
  if (p.test_type) {
    af2.resize((size_t)bsz * P); mac2.resize((size_t)bsz * P); info2.resize((size_t)bsz * P); ns2.resize((size_t)bsz * P);
    af_all2.resize(bsz); mac_all2.resize(bsz); ns_all2.resize(bsz); flags2.resize(bsz);
  }
  rg_s2_out out2{af2.data(), ns2.data(), mac2.data(), af_all2.data(), ns_all2.data(), mac_all2.data(), flags2.data(),
                 scale_fac.data(), stat.data(), beta.data(), se.data(), chisq.data()};
  std::vector<double> res((size_t)N * P), scf(P);
  std::vector<uint8_t> npf;
  int cur_chr = -1;
  size_t n_ignored = 0;
  for (size_t b = b_first; b < blocks.size(); ++b) {
    const int chrom = blocks[b].chrom;
    if (chrom != cur_chr) {
      cur_chr = chrom;
      log << "Chromosome " << chrom << "\n";
      // blup_read_chr + compute_res (src/Step2_Models.cpp:96-124, src/Data.cpp:2386-2404)
      for (int i = 0; i < P; ++i) {
        const std::vector<double> blup = blup_for_chr(locos[i], ss, ph, i, chrom);
        double ssq = 0.0;
        for (int64_t s = 0; s < N; ++s) {
          const double r = (ph.Y[(size_t)i * N + s] - blup[s]) * ph.mask[(size_t)i * N + s];
          res[(size_t)i * N + s] = r;
          ssq += r * r;
        }
        const double psd = std::sqrt(ssq) / std::sqrt(ph.neff[i] - ph.C);
        for (int64_t s = 0; s < N; ++s) res[(size_t)i * N + s] /= psd;
        scf[i] = ph.scale_Y[i] * psd;
      }
      const std::vector<uint8_t> male = male_vector(use_bgen ? gg.sex_file : g.sex_file, sample_idx);
      rg_check(rg_s2_set_sex(h, chrom == 23 ? male.data() : nullptr));
      rg_check(rg_s2_set_chr(h, res.data(), scf.data()));
    }
    pending.get();
    if (b + 1 < blocks.size()) pending = fetch(b + 1);
    if (!use_bgen)
      gc.run(rows[b & 1].data(), (size_t)blocks[b].size * g.row_stride, blocks[b].size, [&](const uint8_t* r, const rg_s2_out* o) {
        rg_check(rg_s2_block_bed(h, r, (int64_t)g.row_stride, blocks[b].size, subset ? sample_idx.data() : nullptr, p.ref_first, 0.0, o));
      });
    if (non_par_flags(p, snps, blocks[b], npf)) rg_check(rg_s2_set_non_par(h, npf.data(), blocks[b].size));
    if (use_bgen) {
      const uint8_t *pd = probs[b & 1].data(), *md = pmiss[b & 1].data();
      if (dev_inflate) rg_check(rg_bgen_inflate(h, comp[b & 1].data(), comp_offs[b & 1].data(), (int64_t)n_file, blocks[b].size, &pd, &md));
      rg_check(rg_s2_block_bgen8(h, pd, md, (int64_t)n_file, blocks[b].size,
                                 subset ? sample_idx.data() : nullptr, p.ref_first, p.min_mac, &out, info.data()));
      if (p.test_type) {
        recode.probs(probs[b & 1].data(), (size_t)blocks[b].size * n_file);
        rg_check(rg_s2_block_bgen8(h, pd, md, (int64_t)n_file, blocks[b].size, subset ? sample_idx.data() : nullptr, p.ref_first,
                                   0.0, &out2, info2.data()));
      }
    } else if (pgen_dev) {
      const uint8_t* drows = nullptr;
      int64_t dstride = 0;
      pgen_rows_device(h, pbatch[b & 1], blocks[b].size, (int64_t)g.pg->n_file, (int)b, &drows, &dstride);
      rg_check(rg_s2_block_bed(h, drows, dstride, blocks[b].size, subset ? sample_idx.data() : nullptr, p.ref_first, p.min_mac, &out));
    } else {
      rg_check(rg_s2_block_bed(h, rows[b & 1].data(), (int64_t)g.row_stride, blocks[b].size,
                               subset ? sample_idx.data() : nullptr, p.ref_first, p.min_mac, &out));
      if (p.test_type) {
        recode.bed(rows[b & 1].data(), (size_t)blocks[b].size * g.row_stride);
        rg_check(rg_s2_block_bed(h, rows[b & 1].data(), (int64_t)g.row_stride, blocks[b].size,
                                 subset ? sample_idx.data() : nullptr, p.ref_first, 0.0, &out2));
      }
    }
    if (p.test_type) merge_recode_flags(blocks[b].size, flags.data(), flags2.data(), af_all2.data());
    for (int v = 0; v < blocks[b].size; ++v) {
      if (flags[v] & 3) { ++n_ignored; continue; }            // no row for ignored variants (split mode)
      if (use_info1 && p.min_info > 0 && info1[b & 1][v] < p.min_info) { ++n_ignored; continue; }
      const Snp& s = snps[blocks[b].first + v];
      head_s.clear();                                        // print_sum_stats_head, src/Step2_Models.cpp:2410-2418
      head_s += std::to_string(s.chrom); head_s += ' ';
      head_s += std::to_string(s.pos); head_s += ' ';
      head_s += s.id; head_s += ' ';
      head_s += s.allele0; head_s += ' ';
      head_s += s.allele1; head_s += ' ';
      if (p.htp) {                                             // print_sum_stats_head_htp :2419-2426
        head_s = s.id + "\t" + std::to_string(s.chrom) + "\t" + std::to_string(s.pos) + "\t" + s.allele0 + "\t" + s.allele1 + "\t";
      }
      if (p.no_split) {                                        // print_sum_stats_all :2441-2493
        long n_rr, n_ra, n_aa;
        if (use_bgen) { n_rr = d_rr[b & 1][v]; n_aa = d_aa[b & 1][v]; n_ra = ns_all[v] - n_rr - n_aa; }
        else gc.counts(v, af_all[v], ns_all[v], n_rr, n_ra, n_aa);
        append_sumstats_all_start(w.obuf_all, head_s, af_all[v], ns_all[v], n_rr, n_ra, n_aa, test_name(p.test_type), use_bgen,
                                  use_bgen ? info1[b & 1][v] : -1.0);
      }
      for (int i = 0; i < P; ++i) {
        const size_t e = (size_t)v * P + i;
        const bool have = !(mac[e] < p.min_mac) &&             // ignored_trait (src/Geno.cpp:3102)
                          !(use_bgen && info[e] < p.min_info);  // --minINFO (src/Geno.cpp:3142-3146)
        if (p.no_split) { append_sumstats_all_trait(w.obuf_all, have, beta[e], se[e], chisq[e], get_logp(chisq[e]), true); continue; }
        if (!have) continue;
        if (p.htp) {
          // print_sum_stats_htp for a quantitative trait.  Genotype counts of the trait's samples (update_genocounts,
          // src/Geno.cpp:2986-3003) counted on the host in the fetch thread (BedTraitCounts / BgenFile::trait_counts).
          // SCORE / SKATV are the numerator and denominator of the statistic (dt_thr->scores / skat_var,
          // src/Step2_Models.cpp:391-394, :421-424): se = scf / sqrt(denum), stat = num / sqrt(denum).
          HtpRow r;
          r.model = htp_model.c_str();
          r.beta = beta[e]; r.se = se[e]; r.chisq = chisq[e]; r.logp = get_logp(chisq[e]); r.af = af[e]; r.mac = mac[e];
          for (int k = 0; k < 3; ++k) r.gc[k] = htp_cnt[b & 1][e * 6 + k];
          if (use_bgen) r.info = info[e];                      // dosages: the trait's INFO
          const double sqrt_den = scf[i] / se[e];
          r.score = stat[e] * sqrt_den; r.skat_var = sqrt_den * sqrt_den;
          append_htp_row(obuf[i], head_s, ph.names[i], p.htp_cohort, r);
          continue;
        }
        append_sumstats_row(obuf[i], head_s, af[e], use_bgen, use_bgen ? info[e] : -1.0, ns[e], test_name(p.test_type), beta[e], se[e], chisq[e],
                            get_logp(chisq[e]), true);   // print_sum_stats_single :2502-2540
      }
      if (p.no_split) w.obuf_all += " NA\n";
    }
    w.flush();
    log << " block [" << b + 1 << "/" << blocks.size() << "] : done\n";
  }
  w.close();
  log << "\nNumber of ignored tests due to low MAC or low variance : " << n_ignored << "\n";
}

// Step 2 for binary traits (--bt [--firth --approx]) on BGEN dosages or .bed hard calls.
// Control flow of Data::test_snps_fast for trait_mode 1 (src/Data.cpp:2230-2383): per chromosome the null
// logistic / null Firth fits (host, O(N C^2)), per block the score test and the Firth fallback (GPU).
void run_step2_bt(const Params& p, Log& log) {
  const bool use_bgen = !p.bgen.empty();
  BedFile gb;
  BgenFile gg;
  const auto excl = read_id_list(p.exclude, 1), extr = read_id_list(p.extract, 1), rem = read_id_list(p.remove, 2),
             keep = read_id_list(p.keep, 2);
  if (use_bgen) {
    gg.sex_specific = p.sex_specific;
    gg.open(p.bgen, p.sample, p.ref_first, excl, extr, rem, keep, p.chrs, p.bgi);
    if (gg.used_bgi) log << "   -index bgi file [" << (p.bgi.empty() ? p.bgen + ".bgi" : p.bgi) << "]\n";
    log << " * bgen                : [" << p.bgen << "] n_snps = " << gg.snps.size() << ", n_samples = " << gg.keys.size() << "\n";
  } else {
    open_rows(p, gb, excl, extr, rem, keep, log);
  }
  apply_range(p, gg.snps);
  apply_range(p, gb.snps);
  if (gb.pg) apply_range(p, gb.pg->snps);
  if (p.set_range && (use_bgen ? gg.snps : gb.snps).empty()) throw Fail("no variant left to include in analysis.");
  const std::vector<Snp>& snps = use_bgen ? gg.snps : gb.snps;
  const std::vector<std::string>& keys = use_bgen ? gg.keys : gb.keys;
  const std::vector<int32_t>& sample_idx = use_bgen ? gg.sample_idx : gb.sample_idx;
  const size_t n_file = use_bgen ? gg.n_file : gb.keys_file.size();
  const SampleSet ss{keys, use_bgen ? gg.key_to_ind : gb.key_to_ind};
  Pheno ph;
  std::vector<Loco> locos;
  load_step2_inputs(p, ss, use_bgen ? gg.ids_file : gb.ids_file, sample_idx, ph, locos, log);
  const int64_t N = ph.N;
  const int P = ph.P, C = ph.C;
  const auto blocks = set_blocks(snps, p.bsize);
  log << " * # blocks            : [" << blocks.size() << "]\n";
  const double z_thr = z_threshold(p.p_thresh);
  // --htp: test_string + wgr_string + correction_type (src/Data.cpp:2075-2102)
  const std::string htp_model = std::string(test_name(p.test_type)) + (p.ignore_pred ? "" : "-WGR") + (p.firth ? "-FIRTH" : p.spa ? "-SPA" : "-LOG");
  if (p.firth) log << " * using approximate Firth correction for logistic regression p-values less than " << p.p_thresh << "\n";
  std::vector<std::string> null_firth_files;                 // check_blup-like list (src/Step2_Models.cpp:1896-1927)
  if (p.firth && !p.null_firth_list.empty()) {
    log << " * reading null Firth estimates using file : [" << p.null_firth_list << "]\n";
    null_firth_files.assign(P, "");
    LineReader fr(p.null_firth_list);
    std::string line;
    std::set<std::string> seen;
    while (fr.getline(line)) {
      const auto t = split_ws(line);
      if (t.empty()) continue;
      if (t.size() != 2) throw Fail("incorrectly formatted blup list file : " + p.null_firth_list);
      const auto it = std::find(ph.names.begin(), ph.names.end(), t[0]);
      if (it == ph.names.end()) continue;                    // unrecognised phenotypes are ignored
      if (!seen.insert(t[0]).second) throw Fail("phenotype '" + t[0] + "' appears more than once in file.");
      { std::ifstream probe_f(t[1]); if (!probe_f) throw Fail("file " + t[1] + " cannot be opened."); }
      null_firth_files[(size_t)(it - ph.names.begin())] = t[1];
    }
  }
  if (p.spa) log << " * using SPA correction for logistic regression p-values less than " << p.p_thresh << "\n";

  rg_step2_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.device = p.gpu; cfg.n_samples = N; cfg.n_cov = C; cfg.n_pheno = P; cfg.max_block_size = p.bsize;
  cfg.n_analyzed = ph.n_analyzed; cfg.strict_mode = ph.strict;
  rg_handle h = nullptr;
  HandleGuard guard{h};
  require_device();
  rg_check(rg_step2_create(&cfg, ph.X.data(), ph.mask.data(), ph.in_analysis.data(), &h));

  S2Writers w;
  w.open(p, ph, use_bgen);
  std::vector<std::string>& obuf = w.obuf;                   // rows of the current block, one buffer per trait
  std::string head_s;
  const int bsz = p.bsize;
  GenoCounts gc(p.no_split, bsz, P, use_bgen ? 0 : gb.row_stride, p.ref_first);
  // --af-cc (update_af_cc / compute_aaf_info, src/Geno.cpp:3069-3075, :3120-3127): a second handle whose sample masks are
  // the cases of each trait returns their allele frequency and count from the same block bytes; controls follow by
  // difference of the (exactly reconstructed) allele sums.
  rg_handle hc = nullptr;
  HandleGuard guard_cases{hc};
  std::vector<double> afc, macc, afc_all, macc_all, statc, betac, sec, chisqc, scalec, infoc;
  std::vector<int32_t> nsc, nsc_all, flagsc;
  if (p.af_cc) {
    std::vector<uint8_t> mask_case(ph.mask.size());
    for (size_t e = 0; e < mask_case.size(); ++e) mask_case[e] = ph.mask[e] && ph.Y_raw[e] == 1.0;
    rg_step2_config cfgc = cfg;
    cfgc.strict_mode = 0;                                    // per-trait masks differ from the analysis set here
    rg_check(rg_step2_create(&cfgc, ph.X.data(), mask_case.data(), ph.in_analysis.data(), &hc));
    const std::vector<double> zero((size_t)N * P, 0.0), one(P, 1.0);
    rg_check(rg_s2_set_chr(hc, zero.data(), one.data()));
    const size_t bp = (size_t)bsz * P;
    afc.resize(bp); macc.resize(bp); statc.resize(bp); betac.resize(bp); sec.resize(bp); chisqc.resize(bp); infoc.resize(bp); nsc.resize(bp);
    afc_all.resize(bsz); macc_all.resize(bsz); scalec.resize(bsz); nsc_all.resize(bsz); flagsc.resize(bsz);
  }
  rg_s2_out outc{afc.data(), nsc.data(), macc.data(), afc_all.data(), nsc_all.data(), macc_all.data(), flagsc.data(),
                 scalec.data(), statc.data(), betac.data(), sec.data(), chisqc.data()};
  const double unit = use_bgen ? 255.0 : 1.0;                // allele sums are multiples of 1 / unit
  const int threads = p.threads > 0 ? p.threads : (int)std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
  std::vector<uint8_t> probs[2], pmiss[2], rows[2];          // fetched one block ahead of the GPU call, like the QT path
  for (int k = 0; k < 2; ++k) {
    if (use_bgen) { probs[k].resize((size_t)bsz * n_file * 2); pmiss[k].resize((size_t)bsz * n_file); }
    else rows[k].resize((size_t)bsz * gb.row_stride);
  }
  const bool use_info1 = use_bgen && (p.min_info > 0 || p.no_split);   // variant-level --minINFO / --no-split, see run_step2_qt
  // --htp on dosages: thresholded genotype counts of the cases and controls of each trait (BgenFile::trait_counts)
  // hard calls: the same by popcounts over the 2-bit rows (BedTraitCounts)
  const bool htp_bgen = use_bgen && p.htp;
  std::vector<uint8_t> htp_cls, htp_npf[2];
  const std::vector<uint8_t> htp_male = p.htp ? male_vector(use_bgen ? gg.sex_file : gb.sex_file, sample_idx) : std::vector<uint8_t>();
  std::vector<long> htp_cnt[2];
  BedTraitCounts btc;
  if (p.htp) {
    htp_cls.resize((size_t)P * N);
    for (size_t e = 0; e < htp_cls.size(); ++e) htp_cls[e] = !ph.mask[e] ? 0 : ph.Y_raw[e] == 1.0 ? 2 : 1;
    for (int k = 0; k < 2; ++k) htp_cnt[k].resize((size_t)bsz * P * 6);
    if (!use_bgen) btc.init(P, true, p.ref_first, n_file, sample_idx, htp_cls.data(), htp_male.data());
  }
  const bool dev_inflate = use_bgen && p.gpu_inflate && gg.compression == 1 && p.test_type == 0 && !use_info1 && !htp_bgen;
  if (use_bgen && p.gpu_inflate)
    log << (dev_inflate ? " * bgen genotype blocks are inflated on the GPU\n"
                        : "   -WARNING: --gpu-inflate needs zlib-compressed payloads, the additive test and no --minINFO / --no-split / --htp; inflating on the host.\n");
  std::vector<uint8_t> comp[2];
  std::vector<uint64_t> comp_offs[2];
  std::vector<double> info1[2];
  std::vector<long> d_rr[2], d_aa[2];
  if (use_info1) for (int k = 0; k < 2; ++k) { info1[k].resize(bsz); d_rr[k].resize(bsz); d_aa[k].resize(bsz); }
  const bool pgen_dev = !use_bgen && gb.pg && pgen_on_device() && !p.no_split && !p.htp && p.test_type == 0 && !hc;   // --htp counts on host rows
  if (pgen_dev) log << " * pgen records are decoded on the GPU\n";
  PgenBatch pbatch[2];
  std::future<void> pending;
  auto fetch = [&](size_t b) {
    return std::async(std::launch::async, [&, b] {
      if (dev_inflate) gg.read_block_compressed(blocks[b].first, blocks[b].size, comp[b & 1], comp_offs[b & 1]);
      else if (use_bgen) {
        gg.read_block(blocks[b].first, blocks[b].size, probs[b & 1].data(), pmiss[b & 1].data(), threads);
        if (use_info1) gg.info_all(probs[b & 1].data(), pmiss[b & 1].data(), blocks[b].size, ph.in_analysis.data(), p.ref_first,
                                   info1[b & 1].data(), threads, d_rr[b & 1].data(), d_aa[b & 1].data());
        if (htp_bgen) {
          const bool np = non_par_flags(p, snps, blocks[b], htp_npf[b & 1]);
          gg.trait_counts(probs[b & 1].data(), pmiss[b & 1].data(), blocks[b].size, htp_cls.data(), P, true, p.ref_first,
                          htp_cnt[b & 1].data(), threads, htp_male.data(), np ? htp_npf[b & 1].data() : nullptr);
        }
      }
      else if (pgen_dev) gb.pg->gather(blocks[b].first, blocks[b].size, pbatch[b & 1]);
      else {
        gb.read_rows(blocks[b].first, blocks[b].size, rows[b & 1].data());
        if (p.htp) {
          const bool np = non_par_flags(p, snps, blocks[b], htp_npf[b & 1]);
          btc.count(rows[b & 1].data(), gb.row_stride, blocks[b].size, np ? htp_npf[b & 1].data() : nullptr, htp_cnt[b & 1].data(), threads);
        }
      }
    });
  };
  if (blocks.empty()) throw Fail("no variant left to include in analysis.");
  if (p.start_block > (int)blocks.size()) throw Fail("Starting block > number of blocks analyzed");   // src/Data.cpp:2863-2864
  const size_t b_first = p.start_block > 1 ? (size_t)p.start_block - 1 : 0;
  if (b_first) log << "    + skipping to block #" << p.start_block << "\n";
  if (!blocks.empty()) pending = fetch(b_first);
  std::vector<double> af((size_t)bsz * P), mac((size_t)bsz * P), stat((size_t)bsz * P), beta((size_t)bsz * P),
      se((size_t)bsz * P), chisq((size_t)bsz * P), info((size_t)bsz * P), af_all(bsz), mac_all(bsz), scale_fac(bsz);
  std::vector<int32_t> ns((size_t)bsz * P), ns_all(bsz), flags(bsz);
  rg_s2_out out{af.data(), ns.data(), mac.data(), af_all.data(), ns_all.data(), mac_all.data(), flags.data(),
                scale_fac.data(), stat.data(), beta.data(), se.data(), chisq.data()};
  const bool subset = keys.size() != n_file;
  const Recode recode(p.test_type, p.ref_first);             // --test dominant / recessive: see run_step2_qt
  std::vector<double> af2, mac2, af_all2, mac_all2, info2;
  std::vector<int32_t> ns2, ns_all2, flags2;
  if (p.test_type) {
    af2.resize((size_t)bsz * P); mac2.resize((size_t)bsz * P); info2.resize((size_t)bsz * P); ns2.resize((size_t)bsz * P);
    af_all2.resize(bsz); mac_all2.resize(bsz); ns_all2.resize(bsz); flags2.resize(bsz);
  }
  rg_s2_out out2{af2.data(), ns2.data(), mac2.data(), af_all2.data(), ns_all2.data(), mac_all2.data(), flags2.data(),
                 scale_fac.data(), stat.data(), beta.data(), se.data(), chisq.data()};
  std::vector<uint8_t> npf;
  int cur_chr = -1;
  size_t n_ignored = 0, n_firth = 0, n_fail = 0;
  for (size_t b = b_first; b < blocks.size(); ++b) {
    const int chrom = blocks[b].chrom, bs = blocks[b].size;
    if (chrom != cur_chr) {
      cur_chr = chrom;
      log << "Chromosome " << chrom << "\n";
      std::vector<double> gsm((size_t)P * N), gs((size_t)P * N), yres((size_t)P * N), xg((size_t)P * C * N), off, yhat;
      if (p.firth) off.resize((size_t)P * N);
      if (p.spa) yhat.resize((size_t)P * N);
      for (int i = 0; i < P; ++i) {
        const std::vector<double> blup = blup_for_chr(locos[i], ss, ph, i, chrom);
        // --use-null-firth: starting values of this chromosome from the Step-1 file (get_beta_start_firth, :1936-1980)
        std::vector<double> fstart;
        if (p.firth && !null_firth_files.empty() && !null_firth_files[i].empty()) {
          LineReader fr(null_firth_files[i]);
          std::string line;
          while (fr.getline(line)) {
            const auto t = split_ws(line);
            if (t.empty()) throw Fail("error reading null firth estimates file");
            if (chr_str_to_int(t[0]) != chrom) continue;
            if ((int)t.size() - 1 > C) throw Fail("file has more predictors than included in analysis (=" + std::to_string(t.size()) + " vs " + std::to_string(C) + ")");
            for (size_t j = 1; j < t.size(); ++j) {
              const double v = convert_double(t[j]);
              if (v == kMissing) throw Fail("no missing values allowed in file");
              fstart.push_back(v);
            }
            break;
          }
        }
        const BtNull nm = fit_bt_null(ph.names[i], &ph.Y_raw[(size_t)i * N], ph.X.data(), N, C, blup.data(),
                                      &ph.mask[(size_t)i * N], p.firth, fstart.empty() ? nullptr : &fstart);
        std::copy(nm.gamma_sqrt_mask.begin(), nm.gamma_sqrt_mask.end(), gsm.begin() + (size_t)i * N);
        std::copy(nm.gamma_sqrt.begin(), nm.gamma_sqrt.end(), gs.begin() + (size_t)i * N);
        std::copy(nm.yres.begin(), nm.yres.end(), yres.begin() + (size_t)i * N);
        std::copy(nm.x_gamma.begin(), nm.x_gamma.end(), xg.begin() + (size_t)i * C * N);
        if (p.firth) std::copy(nm.firth_offset.begin(), nm.firth_offset.end(), off.begin() + (size_t)i * N);
        if (p.spa) std::copy(nm.y_hat_p.begin(), nm.y_hat_p.end(), yhat.begin() + (size_t)i * N);
      }
      const std::vector<uint8_t> male = male_vector(use_bgen ? gg.sex_file : gb.sex_file, sample_idx);
      rg_check(rg_s2_set_sex(h, chrom == 23 ? male.data() : nullptr));
      rg_s2_bt_chr st{gsm.data(), gs.data(), yres.data(), xg.data(), ph.Y_raw.data(), p.firth ? off.data() : nullptr,
                      p.spa ? yhat.data() : nullptr};
      rg_check(rg_s2_set_chr_bt(h, &st));
    }
    pending.get();
    if (b + 1 < blocks.size()) pending = fetch(b + 1);
    if (!use_bgen)
      gc.run(rows[b & 1].data(), (size_t)bs * gb.row_stride, bs, [&](const uint8_t* r, const rg_s2_out* o) {
        rg_check(rg_s2_block_bed_bt(h, r, (int64_t)gb.row_stride, bs, subset ? sample_idx.data() : nullptr, p.ref_first, 0.0, o));
      });
    if (non_par_flags(p, snps, blocks[b], npf)) rg_check(rg_s2_set_non_par(h, npf.data(), bs));
    if (use_bgen) {
      const uint8_t *pd = probs[b & 1].data(), *md = pmiss[b & 1].data();
      if (dev_inflate) rg_check(rg_bgen_inflate(h, comp[b & 1].data(), comp_offs[b & 1].data(), (int64_t)n_file, bs, &pd, &md));
      rg_check(rg_s2_block_bgen8_bt(h, pd, md, (int64_t)n_file, bs,
                                    subset ? sample_idx.data() : nullptr, p.ref_first, p.min_mac, &out, info.data()));
      if (hc) rg_check(rg_s2_block_bgen8(hc, pd, md, (int64_t)n_file, bs, subset ? sample_idx.data() : nullptr, p.ref_first, 0.0,
                                         &outc, infoc.data()));
      if (p.test_type) {
        recode.probs(probs[b & 1].data(), (size_t)bs * n_file);
        rg_check(rg_s2_block_bgen8_bt(h, pd, md, (int64_t)n_file, bs, subset ? sample_idx.data() : nullptr, p.ref_first, 0.0,
                                      &out2, info2.data()));
      }
    } else if (pgen_dev) {
      const uint8_t* drows = nullptr;
      int64_t dstride = 0;
      pgen_rows_device(h, pbatch[b & 1], bs, (int64_t)gb.pg->n_file, (int)b, &drows, &dstride);
      rg_check(rg_s2_block_bed_bt(h, drows, dstride, bs, subset ? sample_idx.data() : nullptr, p.ref_first, p.min_mac, &out));
    } else {
      // hard calls go to the GPU as they are (2 bits per sample)
      rg_check(rg_s2_block_bed_bt(h, rows[b & 1].data(), (int64_t)gb.row_stride, bs, subset ? sample_idx.data() : nullptr,
                                  p.ref_first, p.min_mac, &out));
      if (hc) rg_check(rg_s2_block_bed(hc, rows[b & 1].data(), (int64_t)gb.row_stride, bs, subset ? sample_idx.data() : nullptr,
                                       p.ref_first, 0.0, &outc));
      if (p.test_type) {
        recode.bed(rows[b & 1].data(), (size_t)bs * gb.row_stride);
        rg_check(rg_s2_block_bed_bt(h, rows[b & 1].data(), (int64_t)gb.row_stride, bs, subset ? sample_idx.data() : nullptr,
                                    p.ref_first, 0.0, &out2));
      }
    }
    if (p.test_type) merge_recode_flags(bs, flags.data(), flags2.data(), af_all2.data());
    if (use_info1)                                           // ignored_snp: counts as one ignored variant, no Firth / SPA
      for (int v = 0; v < bs; ++v) if (p.min_info > 0 && info1[b & 1][v] < p.min_info) flags[v] |= 1;
    // Firth fallback for |z| above the --pThresh threshold (check_pval_snp, src/Step2_Models.cpp:1988-2041)
    std::vector<int32_t> sel_v, sel_t, fstatus;
    std::vector<double> fbeta, fse, flrt;
    std::map<std::pair<int, int>, int> fidx;
    std::map<std::pair<int, int>, double> spa_logp;
    if (p.firth || p.spa) {
      for (int v = 0; v < bs; ++v) {
        if (flags[v] & (1 | 16)) continue;
        for (int i = 0; i < P; ++i) {
          const size_t e = (size_t)v * P + i;
          if (mac[e] < p.min_mac || !(std::fabs(stat[e]) > z_thr)) continue;
          fidx[{v, i}] = (int)sel_v.size();
          sel_v.push_back(v); sel_t.push_back(i);
        }
      }
      const size_t nsel = sel_v.size();
      fbeta.resize(nsel); fse.resize(nsel); flrt.resize(nsel); fstatus.resize(nsel);
      if (p.firth) {
        rg_check(rg_s2_firth(h, (int32_t)nsel, sel_v.data(), sel_t.data(), fbeta.data(), fse.data(), flrt.data(), fstatus.data()));
      } else {
        // check_pval_snp, SPA branch (src/Step2_Models.cpp:2021-2029): SE from the score test, beta from the SPA chi-square
        std::vector<double> pv(nsel);
        rg_check(rg_s2_spa(h, (int32_t)nsel, sel_v.data(), sel_t.data(), pv.data(), fstatus.data()));
        for (size_t k = 0; k < nsel; ++k) {
          const size_t e = (size_t)sel_v[k] * P + sel_t[k];
          const double pval = std::max(10.0 * std::numeric_limits<double>::min(), pv[k]);
          flrt[k] = chisq1_from_pvalue(pval);
          fse[k] = se[e];
          fbeta[k] = (beta[e] < 0 ? -1.0 : 1.0) * std::sqrt(flrt[k]) * se[e];
          spa_logp[{sel_v[k], sel_t[k]}] = -std::log10(pval);
        }
      }
      n_firth += nsel;
    }
    for (int v = 0; v < bs; ++v) {
      if (flags[v] & (1 | 16)) { ++n_ignored; continue; }
      const Snp& s = snps[blocks[b].first + v];
      head_s.clear();                                        // print_sum_stats_head, src/Step2_Models.cpp:2410-2418
      head_s += std::to_string(s.chrom); head_s += ' ';
      head_s += std::to_string(s.pos); head_s += ' ';
      head_s += s.id; head_s += ' ';
      head_s += s.allele0; head_s += ' ';
      head_s += s.allele1; head_s += ' ';
      if (p.htp) {                                             // print_sum_stats_head_htp :2419-2426
        head_s = s.id + "\t" + std::to_string(s.chrom) + "\t" + std::to_string(s.pos) + "\t" + s.allele0 + "\t" + s.allele1 + "\t";
      }
      if (p.no_split) {                                        // print_sum_stats_all :2441-2493
        long n_rr, n_ra, n_aa;
        if (use_bgen) { n_rr = d_rr[b & 1][v]; n_aa = d_aa[b & 1][v]; n_ra = ns_all[v] - n_rr - n_aa; }
        else gc.counts(v, af_all[v], ns_all[v], n_rr, n_ra, n_aa);
        append_sumstats_all_start(w.obuf_all, head_s, af_all[v], ns_all[v], n_rr, n_ra, n_aa, test_name(p.test_type), use_bgen,
                                  use_bgen ? info1[b & 1][v] : -1.0);
      }
      for (int i = 0; i < P; ++i) {
        const size_t e = (size_t)v * P + i;
        const bool have = !(mac[e] < p.min_mac) && !(use_bgen && info[e] < p.min_info);   // ignored_trait, --minINFO
        if (!have) {
          if (p.no_split) append_sumstats_all_trait(w.obuf_all, false, 0, 0, 0, 0, false);
          continue;
        }
        double bo = beta[e], so = se[e], co = chisq[e];
        bool pass = true;
        auto f = fidx.find({v, i});
        if (f != fidx.end()) {
          if ((fstatus[f->second] & 15) == 0) { bo = fbeta[f->second]; so = fse[f->second]; co = flrt[f->second]; }
          else { pass = false; ++n_fail; }
        }
        double lp = get_logp(co);
        if (p.spa && pass && f != fidx.end()) lp = spa_logp[{v, i}];   // SPA reports -log10 of its own p-value
        AfCc cc;
        if (hc) {
          const double s_all = std::round(af[e] * 2.0 * ns[e] * unit), s_case = std::round(afc[e] * 2.0 * nsc[e] * unit);
          cc.ns_case = nsc[e];
          cc.ns_control = ns[e] - nsc[e];
          cc.af_case = afc[e];
          cc.af_control = (s_all - s_case) / unit / (2.0 * cc.ns_control);
        }
        if (p.htp) {
          // print_sum_stats_htp for a binary trait (src/Step2_Models.cpp:2542-2646).  Genotype counts of the trait's cases
          // and controls (update_genocounts, src/Geno.cpp:2986-3018) counted on the host in the fetch thread (BedTraitCounts /
          // BgenFile::trait_counts).  SCORE / SKATV (compute_score_bt :523-526, :546): stats * sqrt(denum) with the sign of the minor-allele
          // flip undone, and denum = 1 / se^2 of the score test; cal_factor (check_pval_snp :1993, :2027) = 1 without a
          // correction, stats^2 / corrected chi-square with one.  After a FAILED correction the reference prints whatever
          // cal_factor the thread held before (it returns before the assignment): 1 here.
          HtpRow r;
          r.model = htp_model.c_str(); r.bt = true; r.firth = p.firth;
          r.beta = bo; r.se = so; r.chisq = co; r.logp = lp; r.af = af[e]; r.mac = mac[e]; r.test_pass = pass;
          for (int k = 0; k < 6; ++k) r.gc[k] = htp_cnt[b & 1][e * 6 + k];
          if (use_bgen) r.info = info[e];                      // dosages: the trait's INFO
          const double sqrt_den = 1.0 / se[e];
          r.score = stat[e] * sqrt_den * ((flags[v] & 8) ? -1.0 : 1.0); r.skat_var = sqrt_den * sqrt_den;
          r.cal_factor = (f != fidx.end() && pass) ? (co == 0 ? 0.0 : stat[e] * stat[e] / co) : 1.0;
          append_htp_row(obuf[i], head_s, ph.names[i], p.htp_cohort, r);
          continue;
        }
        if (p.no_split) append_sumstats_all_trait(w.obuf_all, true, bo, so, co, lp, pass);
        else append_sumstats_row(obuf[i], head_s, af[e], use_bgen, use_bgen ? info[e] : -1.0, ns[e], test_name(p.test_type), bo, so, co, lp, pass,
                                 (hc && p.af_cc) ? &cc : nullptr);
      }
      if (p.no_split) w.obuf_all += " NA\n";
    }
    w.flush();
    log << " block [" << b + 1 << "/" << blocks.size() << "] : done\n";
  }
  w.close();
  log << "\nNumber of ignored tests due to low MAC or low variance : " << n_ignored << "\n";
  if (p.firth) log << "Number of tests with Firth correction : " << n_firth << " (" << n_fail << " failed)\n";
  if (p.spa) log << "Number of tests with SPA correction : " << n_firth << " (" << n_fail << " failed)\n";
}

void run_step2(const Params& p_in, Log& log) {
  Params p = p_in;
  if (p.af_cc && (!p.bt || p.no_split)) {                    // src/Regenie.cpp:1076-1079
    log << "WARNING: disabling option --af-cc (only for BTs in step 2 in native output format split by trait).\n";
    p.af_cc = false;
  }
  if (p.htp) p.af_cc = false;                                // HTP rows carry genotype counts, not the --af-cc columns
  if (p.bt) run_step2_bt(p, log); else run_step2_qt(p, log);
}

}  // namespace

int main(int argc, char** argv) {
  Log log;
  // never leave main() while the warm-up thread is still inside the CUDA driver: process exit would tear the runtime
  // down under it (an early input error otherwise hangs at exit)
  struct WarmupJoin {
    ~WarmupJoin() { if (g_ndev.valid()) g_ndev.wait(); }
  } warmup_join;
  try {
    phase("start");
    const Params p = parse_cli(argc, argv);
    log.open(p.out + ".log");
    log << "rgb200 (" << rg_version() << ")\nOptions in effect:\n";
    for (int i = 1; i < argc; ++i) {
      const bool next_is_value = (i + 1 < argc) && !(argv[i + 1][0] == '-' && argv[i + 1][1] == '-');
      log << (argv[i][0] == '-' && argv[i][1] == '-' ? "  " : "") << argv[i] << (next_is_value ? " " : " \\\n");
    }
    log << "\n";
    // CUDA driver initialisation and context creation (of the order of a second on a multi-GPU node) run on a side thread
    // while the text inputs are parsed; a host without any device answers at once and stops here, before touching data
    g_ndev = std::async(std::launch::async, [gpu = p.gpu, G = std::max(1, p.gpus)] {
      const int n = rg_device_count();
      for (int d = 0; d < G && n > 0; ++d) rg_warmup(G > 1 ? d : gpu);
      return n;
    }).share();
    if (g_ndev.wait_for(std::chrono::milliseconds(20)) == std::future_status::ready) require_device();
    phase("rg_device_count");
    const double t0 = now_ms();
    if (p.step == 1) run_step1(p, log); else run_step2(p, log);
    log << "\nElapsed time : " << (now_ms() - t0) / 1e3 << "s\nEnd of rgb200\n";
  } catch (const std::exception& e) {
    log << "ERROR: " << e.what() << "\n";          // same shape as the reference (src/Regenie.cpp:67-92)
    log.close();
    if (g_fast_exit) { fflush(nullptr); _exit(EXIT_FAILURE); }
    return EXIT_FAILURE;
  }
  phase("run finished");
  log.close();
  if (g_fast_exit) { fflush(nullptr); _exit(0); }
  return 0;
}
